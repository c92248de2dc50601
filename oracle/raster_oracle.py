"""f64 NumPy rasteriser following the conventions stated at the top of csrc/raster.cu, with an ambiguity mask.

Conventions: camera-space P = R x + t (the f32 pose and vertices widened to f64); OpenCV projection with skew,
u = fx X/Z + s Y/Z + cx, v = fy Y/Z + cy; pixel (r, c) is sampled at (c + 0.5, r + 0.5); a face covers a sample that
lies inside it or on its boundary, for either winding (no culling), and a face of zero screen area covers nothing; 1/Z
is interpolated with screen-space barycentrics; the nearest fragment wins, and on equal depth the lower face index; a
face with any vertex at Z < znear is dropped whole; a fragment with z < znear or z > zfar is dropped at that pixel;
background depth is 0.  quantize() is the fixed-point window-depth read-back of quantize_bits 16 / 24 / 32.

Ambiguity: an f32 rasteriser may decide a pixel either way when its sample lies within EPS_PX pixels of an edge of a
face that is not behind the winning fragment (or of any face, on background), when the two nearest fragments from
faces that are not exact duplicates lie within EPS_Z (relative) in depth, when the winning depth lies within EPS_Z of
znear or zfar, or when a face covering it has a vertex within EPS_Z of znear.  Every other pixel has one answer, which
the GPU must give exactly in coverage and winning face.
"""
import numpy as np

EPS_PX = 4e-3    # pixels; f32 projection + edge-function error at 640 px is a few 1e-5 px
EPS_Z = 1e-5     # relative depth; f32 1/Z interpolation error is ~1e-6
CHUNK = 1 << 20  # (face, pixel) candidate pairs per vectorised batch


def camera_points(verts, pose):
    """verts [V,3], pose [3,4] -> camera-space points [V,3] f64."""
    pose = np.asarray(pose, np.float64)
    return np.asarray(verts, np.float64) @ pose[:, :3].T + pose[:, 3]


def project(P, K):
    K = np.asarray(K, np.float64)
    u = (K[0, 0] * P[:, 0] + K[0, 1] * P[:, 1]) / P[:, 2] + K[0, 2]
    v = K[1, 1] * P[:, 1] / P[:, 2] + K[1, 2]
    return u, v


def _seg_dist(px, py, ax, ay, bx, by):
    """Distance from points (px, py) to segments a-b (all arrays of one shape)."""
    dx, dy = bx - ax, by - ay
    L2 = dx * dx + dy * dy
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(L2 > 0, ((px - ax) * dx + (py - ay) * dy) / L2, 0.0)
    s = np.clip(s, 0.0, 1.0)
    return np.hypot(px - (ax + s * dx), py - (ay + s * dy))


def rasterize(verts, faces, pose, K, H, W, znear=0.1, zfar=100.0, eps_px=EPS_PX, eps_z=EPS_Z):
    """One render -> dict: depth [H,W] f64 (0 = background), face [H,W] i64 (-1 = background), xyz [H,W,3] f64
    (camera-space point of the winning fragment), ambiguous [H,W] bool."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    P = camera_points(verts, pose)
    u, v = project(P, K)
    Pf = P[faces]
    Zf = Pf[..., 2]
    uf, vf = u[faces], v[faces]
    kept = (Zf >= znear).all(1)
    near_face = (np.abs(Zf - znear) <= eps_z * znear).any(1)       # f32 may drop or keep it
    consider = kept | near_face
    area = (uf[:, 1] - uf[:, 0]) * (vf[:, 2] - vf[:, 0]) - (uf[:, 2] - uf[:, 0]) * (vf[:, 1] - vf[:, 0])
    with np.errstate(invalid="ignore"):
        c0 = np.floor(uf.min(1) - 0.5 - eps_px)
        c1 = np.ceil(uf.max(1) - 0.5 + eps_px)
        r0 = np.floor(vf.min(1) - 0.5 - eps_px)
        r1 = np.ceil(vf.max(1) - 0.5 + eps_px)
    c0, r0 = np.maximum(c0, 0), np.maximum(r0, 0)
    c1, r1 = np.minimum(c1, W - 1), np.minimum(r1, H - 1)
    ok = consider & np.isfinite(c0 + c1 + r0 + r1) & (c1 >= c0) & (r1 >= r0)
    fid = np.nonzero(ok)[0]
    c0, c1, r0, r1 = (a[fid].astype(np.int64) for a in (c0, c1, r0, r1))
    nw = c1 - c0 + 1
    cnt = nw * (r1 - r0 + 1)

    frag_pix, frag_z, frag_f = [], [], []     # covering fragments inside [znear, zfar]
    near_pix, near_z = [], []                 # samples within eps_px of an edge, with the face's depth there
    amb_pix = []                              # unconditionally ambiguous samples
    starts = np.concatenate([[0], np.cumsum(cnt)])
    i = 0
    while i < len(fid):
        j = int(np.searchsorted(starts, starts[i] + CHUNK, side="right")) - 1
        j = max(j, i + 1)
        sl = slice(i, j)
        n_sl = cnt[sl]
        fi = np.repeat(np.arange(i, j), n_sl)
        k = np.arange(int(n_sl.sum())) - np.repeat(starts[i:j] - starts[i], n_sl)
        px = c0[fi] + k % nw[fi]
        py = r0[fi] + k // nw[fi]
        f = fid[fi]
        sx, sy = px + 0.5, py + 0.5
        U, Vv, Z, A = uf[f], vf[f], Zf[f], area[f]
        e0 = (U[:, 1] - sx) * (Vv[:, 2] - sy) - (U[:, 2] - sx) * (Vv[:, 1] - sy)
        e1 = (U[:, 2] - sx) * (Vv[:, 0] - sy) - (U[:, 0] - sx) * (Vv[:, 2] - sy)
        e2 = (U[:, 0] - sx) * (Vv[:, 1] - sy) - (U[:, 1] - sx) * (Vv[:, 0] - sy)
        nz = A != 0
        with np.errstate(invalid="ignore", divide="ignore"):
            w0, w1, w2 = e0 / A, e1 / A, e2 / A
            izp = w0 / Z[:, 0] + w1 / Z[:, 1] + w2 / Z[:, 2]
            zp = 1.0 / izp
        inside = nz & (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
        dist = np.minimum(np.minimum(_seg_dist(sx, sy, U[:, 1], Vv[:, 1], U[:, 2], Vv[:, 2]),
                                     _seg_dist(sx, sy, U[:, 2], Vv[:, 2], U[:, 0], Vv[:, 0])),
                          _seg_dist(sx, sy, U[:, 0], Vv[:, 0], U[:, 1], Vv[:, 1]))
        near = dist <= eps_px
        pix = py * W + px
        fk = kept[f]
        win = inside & fk & (zp >= znear) & (zp <= zfar)
        frag_pix.append(pix[win]); frag_z.append(zp[win]); frag_f.append(f[win])
        # the depth of a nearly-covering face at the sample: its plane, or its nearest vertex when degenerate
        zn = np.where(nz & np.isfinite(zp) & (zp > 0), zp, Z.min(1))
        near_pix.append(pix[near]); near_z.append(zn[near])
        clip = inside & fk & ((np.abs(zp - znear) <= eps_z * znear) | (np.abs(zp - zfar) <= eps_z * zfar))
        amb_pix.append(pix[clip | ((inside | near) & near_face[f])])
        i = j

    pix = np.concatenate(frag_pix) if frag_pix else np.zeros(0, np.int64)
    zs = np.concatenate(frag_z) if frag_z else np.zeros(0)
    fs = np.concatenate(frag_f) if frag_f else np.zeros(0, np.int64)
    depth = np.zeros(H * W)
    face = np.full(H * W, -1, np.int64)
    amb = np.zeros(H * W, bool)
    order = np.lexsort((fs, zs, pix))
    pix, zs, fs = pix[order], zs[order], fs[order]
    first = np.ones(len(pix), bool)
    first[1:] = pix[1:] != pix[:-1]
    wi = np.nonzero(first)[0]
    depth[pix[wi]] = zs[wi]
    face[pix[wi]] = fs[wi]
    # second-nearest fragment: ambiguous when close in depth, unless it is an exact duplicate of the winner
    sec = wi + 1
    has2 = sec < len(pix)
    has2[has2] = pix[sec[has2]] == pix[wi[has2]]
    a, b = wi[has2], sec[has2]
    close = zs[b] - zs[a] <= eps_z * zs[a]
    dup = (Pf[fs[a]] == Pf[fs[b]]).all(axis=(1, 2)) & (zs[b] == zs[a])
    amb[pix[a[close & ~dup]]] = True
    npix = np.concatenate(near_pix) if near_pix else np.zeros(0, np.int64)
    nzs = np.concatenate(near_z) if near_z else np.zeros(0)
    front = (depth[npix] == 0) | (nzs <= depth[npix] * (1 + eps_z))
    amb[npix[front]] = True
    if amb_pix:
        amb[np.concatenate(amb_pix)] = True

    depth = depth.reshape(H, W)
    K = np.asarray(K, np.float64)
    cc, rr = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    Y = (rr - K[1, 2]) / K[1, 1] * depth
    X = (cc - K[0, 2] - K[0, 1] * Y / np.where(depth > 0, depth, 1.0)) / K[0, 0] * depth
    return {"depth": depth, "face": face.reshape(H, W), "xyz": np.stack([X, Y, depth], -1),
            "ambiguous": amb.reshape(H, W)}


def quantize(depth, znear, zfar, bits):
    """Fixed-point window depth d = (1/z - 1/n) / (1/f - 1/n), rounded to `bits` bits, read back as f32 and decoded
    as n f / (n - f) / (d + f / (n - f)) in f64; d == 1 (the cleared buffer) and background decode to 0."""
    depth = np.asarray(depth, np.float64)
    n, f = float(znear), float(zfar)
    with np.errstate(divide="ignore"):
        d = (1.0 / depth - 1.0 / n) / (1.0 / f - 1.0 / n)
    q = float((1 << bits) - 1)
    dq = np.float32(np.floor(d * q + 0.5) / q).astype(np.float64)
    out = (n * f / (n - f)) / (dq + f / (n - f))
    return np.where((depth > 0) & (dq != 1.0), out, 0.0)

