"""fp64 / multiprecision restatement of RANSAC-PnP (csrc/pnp_ransac.cu), one stage at a time, written from the
mathematics rather than from the kernel's arithmetic:

  correspondences  get_out_mask (L1 min-max) + get_img_model_points_with_coords2d (gdrn_evaluator.py:1183-1221) on
                   float32 maps, with the row-major source index of every selected pixel
  p3p_all          every real pose of three points and unit bearings: the quartic in the depth ratio from the resultant
                   of the two distance-ratio equations (mpmath.polyroots), then the depths refined on the law-of-cosines
                   system (mpmath.findroot), so an ill-conditioned quartic cannot leak into the result
  pick_fourth      the solution with the smallest reprojection error at the fourth point
  count_inliers    fp64 reprojection-error counts, with the points whose squared error is within 1e-9 (relative) of thr^2
  refit, cost      scipy least_squares (LM, tolerances 1e-15) over rotation vector + t on an inlier set
  ransac_replay    the kernel's documented algorithm from given samples: hypotheses, first maximum, two refit rounds,
                   the final inlier set
"""
import mpmath
import numpy as np

DPS = 50
BOUNDARY_REL = 1e-9


# ------------------------------------------------------------------------------------------------ correspondences
def correspondences(cx, cy, cz, m, c2d, ext, imH, imW, mask_thr=0.5):
    """One ROI's float32 maps cx, cy, cz, m [hw,hw], c2d [2,hw,hw], ext [3] -> (xyz [N,3] f32, img [N,2] f32,
    src [N] row-major pixel index).  mask normalised by (m - min) / (max - min) (a constant mask gives NaN, so
    nothing is selected); selected where > mask_thr and every |xyz_k| > 1e-4 * extent_k."""
    m32 = np.asarray(m, np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        mn = (m32 - m32.min()) / (m32.max() - m32.min())
    e32 = np.asarray(ext, np.float32)
    half = np.float32(0.5)
    xyz = np.stack([(np.asarray(c, np.float32) - half) * e32[k] for k, c in enumerate((cx, cy, cz))], -1).astype(np.float32)
    lim = np.float32(1e-4) * e32
    sel = (mn > np.float32(mask_thr)) & (np.abs(xyz[..., 0]) > lim[0]) & (np.abs(xyz[..., 1]) > lim[1]) & (np.abs(xyz[..., 2]) > lim[2])
    img = np.stack([np.asarray(c2d[0], np.float32) * np.float32(imW), np.asarray(c2d[1], np.float32) * np.float32(imH)], -1)
    src = np.flatnonzero(sel.reshape(-1))
    return xyz.reshape(-1, 3)[src], img.reshape(-1, 2)[src], src


def bearings(uv, K):
    """Unit bearings K^-1 [u, v, 1] / ||.|| of pixels uv [k,2] as mpmath vectors."""
    with mpmath.workdps(DPS):
        fx, s, cx, fy, cy = (mpmath.mpf(float(K[0, 0])), mpmath.mpf(float(K[0, 1])), mpmath.mpf(float(K[0, 2])),
                             mpmath.mpf(float(K[1, 1])), mpmath.mpf(float(K[1, 2])))
        out = []
        for u, v in np.asarray(uv, np.float64):
            yn = (mpmath.mpf(v) - cy) / fy
            xn = (mpmath.mpf(u) - cx - s * yn) / fx
            nn = mpmath.sqrt(xn * xn + yn * yn + 1)
            out.append([xn / nn, yn / nn, 1 / nn])
        return out


# ------------------------------------------------------------------------------------------------ P3P
def _pmul(a, b):
    out = [mpmath.mpf(0)] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            out[i + j] += x * y
    return out


def _padd(*ps):
    n = max(len(p) for p in ps)
    return [sum((p[i] if i < len(p) else mpmath.mpf(0)) for p in ps) for i in range(n)]


def _pneg(a):
    return [-x for x in a]


def _rigid_from_pairs(Xw, Xc):
    """R, t with Xc_i = R Xw_i + t from three exact point pairs: R = [c1 c2 c1xc2] [w1 w2 w1xw2]^-1 (edges from point 0)."""
    def frame(Q):
        a = [Q[1][k] - Q[0][k] for k in range(3)]
        b = [Q[2][k] - Q[0][k] for k in range(3)]
        c = [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
        return mpmath.matrix([[a[i], b[i], c[i]] for i in range(3)])
    R = frame(Xc) * frame(Xw) ** -1
    t = mpmath.matrix(Xc[0]) - R * mpmath.matrix(Xw[0])
    return R, t


def p3p_all(P, f):
    """All real poses (R [3,3], t [3] as float64) with x_cam = R X + t for world points P [3,3] and unit bearings f (three
    mpmath vectors, or float [3,3]): depths s_i > 0 with |s_i f_i - s_j f_j| = |P_i - P_j|."""
    with mpmath.workdps(DPS):
        Pm = [[mpmath.mpf(float(x)) for x in p] for p in np.asarray(P, np.float64)]
        fm = [[mpmath.mpf(x) for x in v] for v in f]
        dot = lambda a, b: a[0] * b[0] + a[1] * b[1] + a[2] * b[2]
        d2 = lambda a, b: dot([a[k] - b[k] for k in range(3)], [a[k] - b[k] for k in range(3)])
        D01, D02, D12 = d2(Pm[0], Pm[1]), d2(Pm[0], Pm[2]), d2(Pm[1], Pm[2])
        if min(D01, D02, D12) == 0:
            return []
        c01, c02, c12 = dot(fm[0], fm[1]), dot(fm[0], fm[2]), dot(fm[1], fm[2])
        # s1 = u s0, s2 = v s0:  D02 (1 + u^2 - 2u c01) = D01 (1 + v^2 - 2v c02);  D12 (1 + u^2 - 2u c01) = D01 (u^2 + v^2 - 2uv c12)
        # as quadratics in u with coefficients polynomial in v (lowest degree first)
        a1, b1, c1 = [D02], [-2 * c01 * D02], _padd([D02], _pneg(_pmul([D01], [1, -2 * c02, 1])))
        a2, b2, c2 = [D12 - D01], [-2 * c01 * D12, 2 * D01 * c12], [D12, 0, -D01]
        # resultant of two quadratics in u: (a1 c2 - a2 c1)^2 - (a1 b2 - a2 b1)(b1 c2 - b2 c1)
        e = _padd(_pmul(a1, c2), _pneg(_pmul(a2, c1)))
        g = _padd(_pmul(a1, b2), _pneg(_pmul(a2, b1)))
        h = _padd(_pmul(b1, c2), _pneg(_pmul(b2, c1)))
        res = _padd(_pmul(e, e), _pneg(_pmul(g, h)))
        while len(res) > 1 and abs(res[-1]) < mpmath.mpf(10) ** (-DPS + 5) * max(abs(x) for x in res):
            res = res[:-1]
        if len(res) < 2:
            return []
        roots = mpmath.polyroots(list(reversed(res)), maxsteps=200, extraprec=200)
        sols = []
        for r in roots:
            if abs(mpmath.im(r)) > mpmath.mpf(10) ** -12 * max(1, abs(r)):
                continue
            v = mpmath.re(r)
            # u: the roots of the first quadratic that also satisfy the second
            A, B, C = a1[0], b1[0], _peval(c1, v)
            disc = B * B - 4 * A * C
            for u in ((-B + mpmath.sqrt(max(disc, 0))) / (2 * A), (-B - mpmath.sqrt(max(disc, 0))) / (2 * A)):
                q = 1 + u * u - 2 * u * c01
                if not (u > 0 and v > 0 and q > 0):
                    continue
                s0 = mpmath.sqrt(D01 / q)
                s = [s0, u * s0, v * s0]
                pairs = ((0, 1, c01, D01), (0, 2, c02, D02), (1, 2, c12, D12))
                F = lambda x0, x1, x2: [[x0, x1, x2][i] ** 2 + [x0, x1, x2][j] ** 2 - 2 * cc * [x0, x1, x2][i] * [x0, x1, x2][j] - DD
                                        for i, j, cc, DD in pairs]
                if max(abs(y) for y in F(*s)) > mpmath.mpf(10) ** -8 * max(D01, D02, D12):
                    continue      # root of the resultant not shared by both equations at this u
                try:
                    s = list(mpmath.findroot(F, s, tol=mpmath.mpf(10) ** (-2 * DPS + 10), maxsteps=50))
                except (ValueError, ZeroDivisionError):
                    continue
                if min(s) <= 0:
                    continue
                Xc = [[s[k] * fm[k][j] for j in range(3)] for k in range(3)]
                R, t = _rigid_from_pairs(Pm, Xc)
                Rn = np.array([[float(R[i, j]) for j in range(3)] for i in range(3)])
                tn = np.array([float(t[i]) for i in range(3)])
                if not any(np.abs(Rn - Ro).max() < 1e-12 and np.abs(tn - to).max() < 1e-12 for Ro, to in sols):
                    sols.append((Rn, tn))
        return sols


def _peval(p, x):
    return sum(c * x ** i for i, c in enumerate(p))


def pick_fourth(sols, X4, uv4, K):
    """The solution with the smallest squared reprojection error at the fourth correspondence (in front of the camera),
    or None."""
    best, arg = np.inf, None
    for R, t in sols:
        e = reproj_sq(R, t, np.asarray(X4, np.float64)[None], np.asarray(uv4, np.float64)[None], K)[0]
        if e < best:
            best, arg = e, (R, t)
    return arg


# ------------------------------------------------------------------------------------------------ inliers, refit
def project(R, t, X, K):
    """[k,2] pixels and [k] depths of X [k,3] under x_cam = R X + t and K (fp64)."""
    xc = np.asarray(X, np.float64) @ np.asarray(R, np.float64).T + np.asarray(t, np.float64)
    K = np.asarray(K, np.float64)
    z = xc[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[0, 0] * xc[:, 0] / z + K[0, 1] * xc[:, 1] / z + K[0, 2]
        v = K[1, 1] * xc[:, 1] / z + K[1, 2]
    return np.stack([u, v], 1), z


def reproj_sq(R, t, X, uv, K):
    """Squared reprojection error, +inf for points at depth <= 1e-9 (the kernel's `project` rejects those)."""
    p, z = project(R, t, X, K)
    e = ((p - np.asarray(uv, np.float64)) ** 2).sum(1)
    return np.where(z > 1e-9, e, np.inf)


def count_inliers(R, t, X, uv, K, thr):
    """-> (count, flags [k] bool, boundary [k] bool): flags = squared error < thr^2 in fp64 (thr as the float32 the kernel
    receives); boundary = within a relative 1e-9 of thr^2, where fp64 rounding decides."""
    thr2 = float(np.float32(thr)) ** 2
    e = reproj_sq(R, t, X, uv, K)
    flags = e < thr2
    return int(flags.sum()), flags, np.abs(e - thr2) <= BOUNDARY_REL * thr2


def _rotvec_to_mat(w):
    from scipy.spatial.transform import Rotation

    return Rotation.from_rotvec(w).as_matrix()


def cost(R, t, X, uv, K):
    """Sum of squared reprojection errors (the LM objective)."""
    p, _ = project(R, t, X, K)
    return float(((p - np.asarray(uv, np.float64)) ** 2).sum())


def refit(R0, t0, X, uv, K):
    """Levenberg-Marquardt (scipy, tolerances 1e-15) on the reprojection error of X [k,3] / uv [k,2] over rotation vector
    + t, from (R0, t0) -> (R, t)."""
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation

    X = np.asarray(X, np.float64)
    uv = np.asarray(uv, np.float64)

    def resid(x):
        p, _ = project(_rotvec_to_mat(x[:3]), x[3:], X, K)
        return (p - uv).ravel()

    x0 = np.concatenate([Rotation.from_matrix(np.asarray(R0, np.float64)).as_rotvec(), np.asarray(t0, np.float64)])
    r = least_squares(resid, x0, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=20000)
    return _rotvec_to_mat(r.x[:3]), r.x[3:].copy()


def cost_gradient(R, t, X, uv, K, h=1e-7):
    """Central-difference gradient of `cost` over (rotation vector perturbation on the left, t): zero at a minimiser."""
    g = np.zeros(6)
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        Rp, Rm = _rotvec_to_mat(d[:3]) @ R, _rotvec_to_mat(-d[:3]) @ R
        g[k] = (cost(Rp, t + d[3:], X, uv, K) - cost(Rm, t - d[3:], X, uv, K)) / (2 * h)
    return g


# ------------------------------------------------------------------------------------------------ the whole algorithm
def hypothesis(X, uv, K, ids):
    """pick_fourth(p3p_all(...)) for the four correspondence ids; None when two ids coincide or no pose exists."""
    if len(set(int(i) for i in ids)) < 4:
        return None
    f = bearings(uv[list(ids[:3])], K)
    return pick_fourth(p3p_all(X[list(ids[:3])], f), X[ids[3]], uv[ids[3]], K)


def ransac_replay(X, uv, K, samples, thr=3.0):
    """The kernel's algorithm from given samples [iters, 4] (ids into X / uv): hypotheses, fp64 counts, best = first
    maximum, then two rounds of (inliers at the pose -> refit on them) and the final inlier set.  Returns a dict with
    hyps, cnt (-1 no model), best, rounds [(flags, start (R, t), end (R, t))], pose (R, t) or None (the -100 sentinel),
    flags and n_inliers."""
    X = np.asarray(X, np.float64)
    uv = np.asarray(uv, np.float64)
    out = dict(hyps=[], cnt=[], best=-1, rounds=[], pose=None, flags=np.zeros(len(X), bool), n_inliers=0)
    if len(X) < 4:
        return out
    for ids in samples:
        h = hypothesis(X, uv, K, ids)
        out["hyps"].append(h)
        out["cnt"].append(-1 if h is None else count_inliers(h[0], h[1], X, uv, K, thr)[0])
    cnt = np.array(out["cnt"])
    best = int(np.argmax(cnt))            # first maximum
    out["best"] = best
    if cnt[best] < 4:
        return out
    R, t = out["hyps"][best]
    for _ in range(2):
        flags = count_inliers(R, t, X, uv, K, thr)[1]
        R1, t1 = refit(R, t, X[flags], uv[flags], K)
        out["rounds"].append((flags, (R, t), (R1, t1)))
        R, t = R1, t1
    out["pose"] = (R, t)
    out["n_inliers"], out["flags"], _ = count_inliers(R, t, X, uv, K, thr)
    return out
