"""The rasteriser (csrc/raster.cu: rast_tri_multi_kernel, rast_resolve_kernel, rast_shade_kernel, rast_clear_kernel)
against oracle/raster_oracle.py, an f64 NumPy rasteriser of the conventions stated at the top of raster.cu, at the scale
BOP evaluation renders: 640 x 480 images, the LM / LMO and YCB-V intrinsics and one K with skew, models in millimetres
0.3 m to 2 m away with up to 20 k faces.

The oracle marks as ambiguous the pixels an f32 rasteriser may decide either way (a sample within EPS_PX of an edge of a
face in front, two nearest fragments within EPS_Z in depth, a depth within EPS_Z of a clip plane).  On every other pixel
coverage and the winning face (the tri_ids of rast_render_meshes_rgb) must equal the oracle's exactly, and depth and the
back-projected xyz_cam must lie within the bars below.  Watertightness is checked without the mask: every pixel inside a
tessellated silhouette must be covered, at the analytic depth.

Each bar is at most 4x the largest error measured on an H100 (80GB HBM3, 700 W power limit) over all cases of the
quantity; the measured maxima and where they occurred are listed next to the bars in BARS.  The CPU tests pin the oracle
itself to hand-worked cases.
"""
import numpy as np
import pytest

from oracle import ops_oracle as OO
from oracle import raster_oracle as RO
from oracle.flat_shade_oracle import flat_shade

H, W = 480, 640
K_LM = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])
K_YCBV = np.array([[1066.778, 0.0, 312.9869], [0.0, 1067.487, 241.3109], [0.0, 0.0, 1.0]])
K_SKEW = np.array([[600.0, 14.0, 318.3], [0.0, 605.0, 236.7], [0.0, 0.0, 1.0]])
KS = {"lm": K_LM, "ycbv": K_YCBV, "skew": K_SKEW}
ZNEAR, ZFAR = 10.0, 10000.0      # mm

# quantity -> bar, with the largest error measured over all cases (H100 80GB HBM3, 700 W power limit) and where
BARS = {
    "depth": 1.6e-5,        # 4.47e-6  ico5 LM at 450 mm; relative |z - z64| / z64 on unambiguous pixels
    "xyz": 1.6e-5,          # 4.47e-6  ico5 LM at 450 mm; |xyz - xyz64| / z64, the skew term of the back-projection included
    "depth_sliver": 3e-5,   # 7.58e-6  slivers LM at 500 mm (the sliver and sub-pixel mesh)
    "xyz_sliver": 3e-5,     # 7.58e-6  slivers LM at 500 mm
    "plane_depth": 8e-7,    # 2.05e-7  tilted grid; relative, tessellated planes against the analytic ray-plane depth
    "quant": 3.0,           # 0.753    32 bits, planes 100 / 3000 mm, 400 mm; |z - decode(z32)| in units of
                            #          z^2 |1/n - 1/f| (2^-bits + 2^-24), the depth step of one LSB
    "rgb": 1,               # 0.501    vertex colours, skew K; u8 levels against the unrounded f64 flat shade
    "refine_t": 2.4e-4,     # 6.1e-5   ROI 1; mm, depth refine translation against the numpy renderer's loop
}
MEASURED = {}


def _note(what, value, case):
    if value > MEASURED.get(what, (-1.0, None))[0]:
        MEASURED[what] = (float(value), case)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, (v, case) in sorted(MEASURED.items()):
        print(f"measured {k}: {v:.3g} at {case}")


# ------------------------------------------------------------------------------------------------ meshes and poses
def _ellipsoid(subdiv, extent_mm):
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    v, f = make_icosphere_mesh(subdiv, extent_mm)
    return np.asarray(v, np.float32), np.asarray(f, np.int32)


def _pyramid():
    """An open four-sided pyramid of four large faces, 900 mm across and 150 mm deep, apex toward the camera."""
    v = np.array([[-450, -450, 0], [450, -450, 0], [450, 450, 0], [-450, 450, 0], [20, -10, -150]], np.float32)
    return v, np.array([[0, 1, 4], [1, 2, 4], [2, 3, 4], [3, 0, 4]], np.int32)


def _slivers(seed=3):
    """Sub-pixel faces (0.1 - 1 mm) and long slivers (50 - 200 mm by 0.001 - 0.05 mm) in a 200 mm box."""
    rs = np.random.RandomState(seed)
    tris = []
    for _ in range(1500):
        c = rs.uniform(-100, 100, 3)
        tris.append(c + rs.uniform(-1, 1, (3, 3)) * rs.uniform(0.1, 1.0))
    for _ in range(300):
        a = rs.uniform(-100, 100, 3)
        d = rs.randn(3); d /= np.linalg.norm(d)
        b = a + d * rs.uniform(50, 200)
        side = np.cross(d, rs.randn(3)); side /= np.linalg.norm(side)
        tris.append(np.stack([a, b, a + 0.5 * (b - a) + side * rs.uniform(0.001, 0.05)]))
    v = np.concatenate(tris).astype(np.float32)
    return v, np.arange(len(v), dtype=np.int32).reshape(-1, 3)


def _rot(seed):
    q, r = np.linalg.qr(np.random.RandomState(seed).randn(3, 3))
    q *= np.sign(np.diag(r))
    return q * np.linalg.det(q)


def _pose(R, t):
    return np.hstack([np.asarray(R, np.float64), np.asarray(t, np.float64).reshape(3, 1)]).astype(np.float32)


def _at_pixel(K, u, v, z):
    """Translation that puts the model origin at pixel (u, v), depth z."""
    y = (v - K[1, 2]) / K[1, 1] * z
    return np.array([(u - K[0, 2] - K[0, 1] * y / z) / K[0, 0] * z, y, z])


MESHES = {"ico4": lambda: _ellipsoid(4, (120.0, 90.0, 100.0)), "ico5": lambda: _ellipsoid(5, (200.0, 160.0, 180.0)),
          "pyramid": _pyramid, "slivers": _slivers}
DISTANCES = {"ico4": (300.0, 900.0, 2000.0), "ico5": (450.0, 1200.0), "pyramid": (700.0, 1000.0, 2000.0),
             "slivers": (500.0, 1300.0)}


# ------------------------------------------------------------------------------------------------ GPU helpers
_MODELS = {}


def _model(dev, key, v, f, colors=None):
    """Each mesh is uploaded once per process (the registry is append-only)."""
    from gdrnpp_bop2022_b200.renderer import Model3D

    if key not in _MODELS:
        _MODELS[key] = Model3D(v, f, device=dev, colors=colors)
    return _MODELS[key]


def _gpu(dev, mesh_ids, poses, Ks, h=H, w=W, znear=ZNEAR, zfar=ZFAR):
    """Both entry points on one batch -> depth, tri_ids, xyz (numpy); the rgb entry point's depth must equal the float
    path bit for bit."""
    import torch

    from gdrnpp_bop2022_b200.renderer import render_meshes, render_meshes_rgb

    ids = torch.as_tensor(np.asarray(mesh_ids, np.int32)).to(dev)
    P = torch.from_numpy(np.asarray(poses, np.float32)).to(dev)
    Kt = torch.from_numpy(np.asarray(Ks, np.float32)).to(dev)
    _, d_rgb, tri = render_meshes_rgb(ids, P, Kt, h, w, znear, zfar, return_tri_ids=True)
    d, xyz = render_meshes(ids, P, Kt, h, w, znear, zfar, return_xyz=True)
    torch.cuda.synchronize()
    d, d_rgb = d.cpu().numpy(), d_rgb.cpu().numpy()
    assert np.array_equal(d.view(np.int32), d_rgb.view(np.int32))
    return d, tri.cpu().numpy(), xyz.cpu().numpy()


def _oracle(v, f, pose, K, h=H, w=W, znear=ZNEAR, zfar=ZFAR):
    return RO.rasterize(v, f, pose, np.asarray(K, np.float32), h, w, znear, zfar)


def _compare(d, tri, xyz, ref, case, min_clear=0, sliver=False):
    """Unambiguous pixels: coverage and winning face exact, depth and xyz within the bars."""
    ok = ~ref["ambiguous"]
    bad = ok & (tri != ref["face"])
    assert not bad.any(), (case, int(bad.sum()), np.argwhere(bad)[:5].tolist())
    cov = ok & (ref["face"] >= 0)
    assert cov.sum() >= min_clear, (case, int(cov.sum()))
    assert (d[ref["face"] < 0][ok[ref["face"] < 0]] == 0).all(), case
    if cov.any():
        z = ref["depth"][cov]
        e_d = (np.abs(d[cov] - z) / z).max()
        e_x = (np.abs(xyz[cov] - ref["xyz"][cov]).max(1) / z).max()
        qd, qx = ("depth_sliver", "xyz_sliver") if sliver else ("depth", "xyz")
        _note(qd, e_d, case); _note(qx, e_x, case)
        assert e_d <= BARS[qd], (case, e_d)
        assert e_x <= BARS[qx], (case, e_x)
    return ok


# ------------------------------------------------------------------------------------------------ CPU: the oracle
def test_oracle_plane_matches_analytic_depth():
    """A tilted two-triangle plane over the whole window renders to the ray-plane depth, with xyz on the rays."""
    K = np.array([[500.0, 7.0, 33.3], [0.0, 510.0, 29.9], [0.0, 0.0, 1.0]], np.float32)
    n_pl, d_pl = np.array([0.2, -0.1, 1.0]), 800.0
    corners = []
    for (c, r) in ((-20, -20), (90, -20), (90, 90), (-20, 90)):
        y = (r - K[1, 2]) / K[1, 1]
        ray = np.array([(c - K[0, 2] - K[0, 1] * y) / K[0, 0], y, 1.0])
        corners.append(ray * d_pl / (ray @ n_pl))
    v = np.array(corners, np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    pose = _pose(np.eye(3), np.zeros(3))
    ref = RO.rasterize(v, f, pose, K, 64, 64, 10.0, 5000.0)
    cc, rr = np.meshgrid(np.arange(64) + 0.5, np.arange(64) + 0.5)
    y = (rr - K[1, 2]) / K[1, 1]
    rays = np.stack([(cc - K[0, 2] - K[0, 1] * y) / K[0, 0], y, np.ones_like(cc)], -1)
    assert (ref["face"] >= 0).all()
    z = np.zeros((64, 64))
    for k, (a, b, c) in enumerate(v.astype(np.float64)[f]):   # the f32 corners make the two faces' planes differ
        n64 = np.cross(b - a, c - a)
        z = np.where(ref["face"] == k, (n64 @ a) / (rays @ n64), z)
    assert np.abs(ref["depth"] - z).max() < 1e-9 * z.max()
    assert np.abs(ref["xyz"] - rays * z[..., None]).max() < 1e-9 * z.max()
    assert ref["ambiguous"].sum() < 64 * 2        # only the samples on the diagonal shared edge
    assert np.array_equal(OO.render_depth(v, f, pose, K, 64, 64, 10.0, 5000.0) > 0, ref["depth"] > 0)


def test_oracle_hand_worked_triangle():
    """Screen triangle (1,1) (5,1) (1,5) at Z = 100: the samples (c+.5, r+.5) with c, r >= 1, c + r <= 5 are covered,
    the hypotenuse included; the samples on it are ambiguous, the others are not."""
    K = np.array([[100.0, 0.0, 0.0], [0.0, 100.0, 0.0], [0.0, 0.0, 1.0]], np.float32)
    v = np.array([[1, 1, 100], [5, 1, 100], [1, 5, 100]], np.float32)   # u = X, v = Y at Z = 100
    ref = RO.rasterize(v, np.array([[0, 1, 2]]), _pose(np.eye(3), np.zeros(3)), K, 8, 8, 1.0, 1000.0)
    cc, rr = np.meshgrid(np.arange(8) + 0.5, np.arange(8) + 0.5)
    inside = (cc >= 1) & (rr >= 1) & (cc + rr <= 6)
    assert np.array_equal(ref["face"] >= 0, inside)
    on_edge = inside & (cc + rr == 6)
    assert ref["ambiguous"][on_edge].all() and not ref["ambiguous"][inside & ~on_edge].any()
    assert np.abs(ref["depth"][inside] - 100.0).max() < 1e-12


def test_oracle_tie_break_and_clip_rules():
    K = np.array([[100.0, 0.0, 4.0], [0.0, 100.0, 4.0], [0.0, 0.0, 1.0]], np.float32)
    pose = _pose(np.eye(3), np.zeros(3))
    quad = np.array([[-1, -1, 20], [1, -1, 20], [1, 1, 20], [-1, 1, 20]], np.float32)
    # exact duplicates (other vertex copies): the lower face index wins, and that is not ambiguous
    v = np.concatenate([quad, quad])
    f = np.array([[4, 5, 6], [4, 6, 7], [0, 1, 2], [0, 2, 3]])
    ref = RO.rasterize(v, f, pose, K, 8, 8, 1.0, 100.0)
    clear = ~ref["ambiguous"]
    assert (ref["face"][clear] >= 0).all() and (ref["face"][clear] <= 1).all() and clear.sum() > 30
    # a nearer copy 1e-3 in front wins whatever its index; 1e-7 in front is ambiguous
    for dz, amb in ((1e-3, False), (1e-7, True)):
        v2 = np.concatenate([quad - np.array([0, 0, dz * 20], np.float32), quad])   # faces 2, 3 nearer
        ref = RO.rasterize(v2, f, pose, K, 8, 8, 1.0, 100.0)
        inner = ref["face"] >= 0
        if amb:
            assert ref["ambiguous"][inner].all()
        else:
            assert set(np.unique(ref["face"][inner & ~ref["ambiguous"]])) == {2, 3}
    # znear drops the whole face, zfar drops the fragment
    tilt = np.array([[-1, -1, 5], [1, -1, 5], [1, 1, 15], [-1, 1, 15]], np.float32)
    ref = RO.rasterize(tilt, np.array([[0, 1, 2], [0, 2, 3]]), pose, K, 8, 8, 6.0, 100.0)
    assert (ref["face"] < 0).all()
    ref = RO.rasterize(tilt, np.array([[0, 1, 2], [0, 2, 3]]), pose, K, 8, 8, 1.0, 9.0)
    cov = ref["face"] >= 0
    assert cov.any() and (~cov).any() and (ref["depth"][cov] <= 9.0).all()
    # the fixed-point decode: 2^bits levels between the planes, d == 1 decodes to 0
    z = np.array([100.0, 1000.0, 9999.9999])
    for bits in (16, 24, 32):
        dq = RO.quantize(z, 10.0, 10000.0, bits)
        step = z ** 2 * (1 / 10.0 - 1 / 10000.0) * (2.0 ** -bits + 2.0 ** -24)
        assert (np.abs(dq[:2] - z[:2]) <= step[:2]).all(), bits
    assert RO.quantize(np.array([10000.0]), 10.0, 10000.0, 16)[0] == 0.0


# ------------------------------------------------------------------------------------------------ GPU: BOP scale
@pytest.mark.gpu
@pytest.mark.parametrize("kname", list(KS))
@pytest.mark.parametrize("mesh", list(MESHES))
def test_bop_scale_depth_and_visibility(dev, mesh, kname):
    v, f = MESHES[mesh]()
    K = KS[kname]
    m = _model(dev, mesh, v, f)
    poses = []
    for i, z in enumerate(DISTANCES[mesh]):
        u0, v0 = (W * (0.35 + 0.15 * i), H * (0.4 + 0.1 * i))
        poses.append(_pose(_rot(10 * i + len(mesh)), _at_pixel(K, u0, v0, z)))
    d, tri, xyz = _gpu(dev, [m.mesh_id] * len(poses), poses, [K] * len(poses))
    for i, pose in enumerate(poses):
        ref = _oracle(v, f, pose, K)
        _compare(d[i], tri[i], xyz[i], ref, (mesh, kname, DISTANCES[mesh][i]), min_clear=20 if mesh == "slivers" else 500,
                 sliver=mesh == "slivers")


def _clip_case(name):
    """-> (verts, faces, pose, znear, zfar, expect_empty)."""
    K = K_LM
    v, f = _ellipsoid(4, (120.0, 90.0, 100.0))
    R = _rot(7)
    border = {"left": (0.0, 240.0), "right": (640.0, 250.0), "top": (300.0, 0.0), "bottom": (330.0, 480.0),
              "corner": (640.0, 480.0)}
    if name in border:
        return v, f, _pose(R, _at_pixel(K, *border[name], 700.0)), ZNEAR, ZFAR, False
    if name == "offscreen":
        return v, f, _pose(R, _at_pixel(K, -120.0, 240.0, 700.0)), ZNEAR, ZFAR, True
    if name == "behind":
        return v, f, _pose(R, np.array([0.0, 0.0, -700.0])), ZNEAR, ZFAR, True
    if name in ("znear", "zfar"):   # a tessellated strip running away from the camera, Z from 60 to 1500 mm
        gx, gz = np.meshgrid(np.linspace(-150, 150, 13), np.linspace(60, 1500, 41))
        pv = np.stack([gx, 0.25 * gz - 60.0, gz], -1).reshape(-1, 3).astype(np.float32)
        quads = [(j * 13 + i, j * 13 + i + 1, (j + 1) * 13 + i + 1, (j + 1) * 13 + i) for j in range(40) for i in range(12)]
        pf = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))], np.int32)
        if name == "znear":   # the near plane cuts faces of the strip: they vanish whole
            return pv, pf, _pose(np.eye(3), np.zeros(3)), 200.0 + 1.7, ZFAR, False
        return pv, pf, _pose(np.eye(3), np.zeros(3)), ZNEAR, 900.0 + 1.3, False
    if name == "degenerate":   # zero-area and collinear faces in front of the object
        a, b = np.array([-60.0, -30.0, -200.0]), np.array([70.0, 40.0, -200.0])
        extra = np.stack([a, b, 0.3 * a + 0.7 * b, a + [0, 0, 1e-3]]).astype(np.float32)
        n0 = len(v)
        v2 = np.concatenate([v, extra])
        f2 = np.concatenate([np.array([[n0, n0, n0 + 1], [n0, n0 + 1, n0 + 2], [n0 + 1, n0, n0], [n0 + 2, n0 + 2, n0 + 2]],
                                      np.int32), f])
        return v2, f2, _pose(R, _at_pixel(K, 320.0, 240.0, 800.0)), ZNEAR, ZFAR, False
    if name == "reversed":
        return v, f[:, ::-1].copy(), _pose(R, _at_pixel(K, 300.0, 220.0, 600.0)), ZNEAR, ZFAR, False
    if name == "duplicated":   # a second copy of every face with other vertex copies: the first copy always wins
        v2 = np.concatenate([v, v])
        f2 = np.concatenate([f + len(v), f])
        return v2, f2, _pose(R, _at_pixel(K, 300.0, 220.0, 600.0)), ZNEAR, ZFAR, False
    raise KeyError(name)


CLIP_CASES = ("left", "right", "top", "bottom", "corner", "offscreen", "behind", "znear", "zfar", "degenerate", "reversed",
              "duplicated")


@pytest.mark.gpu
@pytest.mark.parametrize("name", CLIP_CASES)
def test_clipping_and_border_edges(dev, name):
    v, f, pose, zn, zf, empty = _clip_case(name)
    m = _model(dev, "clip_" + name, v, f)
    d, tri, xyz = _gpu(dev, [m.mesh_id], [pose], [K_LM], znear=zn, zfar=zf)
    ref = _oracle(v, f, pose, K_LM, znear=zn, zfar=zf)
    if empty:
        assert (ref["face"] < 0).all() and (tri[0] < 0).all() and (d[0] == 0).all()
        return
    ok = _compare(d[0], tri[0], xyz[0], ref, name, min_clear=500)
    if name == "duplicated":
        assert (tri[0][tri[0] >= 0] < len(f) // 2).all()
    if name == "znear":   # the faces the plane cuts leave a band of background between the kept faces and the image edge
        P = RO.camera_points(v, pose)
        cut = (P[f][..., 2] < zn).any(1) & (P[f][..., 2] >= zn).any(1)
        assert cut.any()
        # a renderer that clipped per pixel would draw these faces' parts beyond znear
        clipped = OO.render_depth(v, f[cut], pose, K_LM.astype(np.float32), H, W, 1.0, zf)
        band = ok & (ref["face"] < 0) & (clipped >= zn)
        assert band.sum() > 100 and (tri[0][band] < 0).all()
    if name == "zfar":   # the fragments beyond zfar are dropped, the rest of their faces drawn
        beyond = ok & (OO.render_depth(v, f, pose, K_LM.astype(np.float32), H, W, zn, 1e5) > zf)
        assert beyond.sum() > 100 and (tri[0][beyond] < 0).all() and (d[0] <= zf).all()


# ------------------------------------------------------------------------------------------------ GPU: watertightness
def _grid_plane(step=3, n=60, u0=100, v0=100, z=1024.0, fx=512.0, cx=320.0, cy=240.0, seed=0):
    """A fronto-parallel plane at Z = z whose vertices project to pixel centres (fx / z a power of two: exact in f32),
    split into triangles along alternating diagonals, each face's vertex order rotated and flipped at random, so every
    shared edge and vertex passes through pixel centres."""
    rs = np.random.RandomState(seed)
    gi, gj = np.meshgrid(np.arange(n + 1), np.arange(n + 1))
    uu, vv = u0 + 0.5 + step * gi.ravel(), v0 + 0.5 + step * gj.ravel()
    verts = np.stack([(uu - cx) * z / fx, (vv - cy) * z / fx, np.full(uu.shape, z)], -1).astype(np.float32)
    idx = lambda i, j: j * (n + 1) + i
    faces = []
    for j in range(n):
        for i in range(n):
            a, b, c, d = idx(i, j), idx(i + 1, j), idx(i + 1, j + 1), idx(i, j + 1)
            faces += [(a, b, c), (a, c, d)] if (i + j) % 2 else [(a, b, d), (b, c, d)]
    faces = np.array(faces, np.int32)
    for k in range(len(faces)):
        faces[k] = np.roll(faces[k], rs.randint(3))
        if rs.rand() < 0.5:
            faces[k] = faces[k][::-1]
    inner = (slice(v0 + 1, v0 + step * n), slice(u0 + 1, u0 + step * n))
    return verts, faces, inner


def _fan(z=1024.0, fx=512.0, cx=320.0, cy=240.0):
    """A 24-triangle fan around the vertex at pixel centre (320.5, 240.5), rim vertices at pixel centres."""
    ang = np.linspace(0, 2 * np.pi, 25)[:-1]
    rim = np.stack([np.round(40 * np.cos(ang)), np.round(33 * np.sin(ang))], -1) + [320.5, 240.5]
    uv = np.concatenate([[[320.5, 240.5]], rim])
    verts = np.stack([(uv[:, 0] - cx) * z / fx, (uv[:, 1] - cy) * z / fx, np.full(len(uv), z)], -1).astype(np.float32)
    faces = np.array([(0, 1 + k, 1 + (k + 1) % 24) for k in range(24)], np.int32)
    return verts, faces


@pytest.mark.gpu
def test_watertight_tessellations(dev):
    K = np.array([[512.0, 0.0, 320.0], [0.0, 512.0, 240.0], [0.0, 0.0, 1.0]])
    eye = _pose(np.eye(3), np.zeros(3))
    gv, gf, inner = _grid_plane()
    fv, ff = _fan()
    # the same grid tilted (vertices no longer on pixel centres): depth against the analytic plane
    R = np.array([[1, 0, 0], [0, np.cos(0.5), -np.sin(0.5)], [0, np.sin(0.5), np.cos(0.5)]])
    c = gv.astype(np.float64).mean(0)
    tilt = _pose(R, c - R @ c)
    mg, mf = _model(dev, "grid", gv, gf), _model(dev, "fan", fv, ff)
    d, tri, _ = _gpu(dev, [mg.mesh_id, mf.mesh_id, mg.mesh_id], [eye, eye, tilt], [K] * 3)
    # fronto-parallel: every sample inside the grid and the fan is covered, at depth 1024
    assert (tri[0][inner] >= 0).all(), int((tri[0][inner] < 0).sum())
    e = np.abs(d[0][inner] / 1024.0 - 1.0).max()
    _note("plane_depth", e, "grid")
    assert e <= BARS["plane_depth"], e
    fan_ref = _oracle(fv, ff, eye, K)
    inside = fan_ref["face"] >= 0
    assert inside[240, 320] and (tri[1][inside] >= 0).all()
    e = np.abs(d[1][inside] / 1024.0 - 1.0).max()
    _note("plane_depth", e, "fan")
    assert e <= BARS["plane_depth"], e
    assert (tri[1][~inside & ~fan_ref["ambiguous"]] < 0).all()
    # tilted: inside the silhouette (all 3x3 neighbours covered in f64) covered at the ray-plane depth
    ref = _oracle(gv, gf, tilt, K)
    cov = ref["face"] >= 0
    interior = cov.copy()
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            interior &= np.roll(np.roll(cov, dy, 0), dx, 1)
    assert interior.sum() > 20000 and (tri[2][interior] >= 0).all()
    P = RO.camera_points(gv, tilt)
    nrm = np.cross(P[1] - P[0], P[gv.shape[0] - 1] - P[0])
    cc, rr = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    rays = np.stack([(cc - K[0, 2]) / K[0, 0], (rr - K[1, 2]) / K[1, 1], np.ones_like(cc)], -1)
    z = (nrm @ P[0]) / (rays @ nrm)
    e = (np.abs(d[2][interior] - z[interior]) / z[interior]).max()
    _note("plane_depth", e, "tilted grid")
    assert e <= BARS["plane_depth"], e


@pytest.mark.gpu
def test_closed_mesh_shows_no_back_face(dev):
    """A closed 20 k-face ellipsoid filling much of a YCB-V image: inside the silhouette every pixel is covered at the
    front surface's depth, ambiguous pixels included (a crack would show the back surface, 100+ mm deeper)."""
    v, f = MESHES["ico5"]()
    m = _model(dev, "ico5", v, f)
    pose = _pose(_rot(21), _at_pixel(K_YCBV, 330.0, 230.0, 700.0))
    d, tri, xyz = _gpu(dev, [m.mesh_id], [pose], [K_YCBV])
    ref = _oracle(v, f, pose, K_YCBV)
    cov = ref["face"] >= 0
    interior = cov.copy()
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            interior &= np.roll(np.roll(cov, dy, 0), dx, 1)
    assert interior.sum() > 50000
    assert (tri[0][interior] >= 0).all()
    assert (np.abs(d[0][interior] - ref["depth"][interior]) / ref["depth"][interior]).max() <= BARS["depth"]
    _compare(d[0], tri[0], xyz[0], ref, "closed ico5")


# ------------------------------------------------------------------------------------------------ GPU: quantised decode
@pytest.mark.gpu
@pytest.mark.parametrize("bits", (16, 24, 32))
@pytest.mark.parametrize("planes", ((10.0, 10000.0), (100.0, 3000.0)))
def test_quantised_decode_bop_scale(dev, bits, planes):
    """quantize_bits: the decode of the render's own f32 depth to the f64 formula within the bar, and the end result
    within the depth bar plus one LSB's depth step of the f64 render's decode."""
    import torch

    from gdrnpp_bop2022_b200.renderer import render_meshes

    zn, zf = planes
    v, f = MESHES["ico4"]()
    m = _model(dev, "ico4", v, f)
    poses = [_pose(_rot(31), _at_pixel(K_LM, 300.0, 250.0, z)) for z in (400.0, 1000.0, 2500.0)]
    ids = torch.full((3,), m.mesh_id, dtype=torch.int32, device=dev)
    P = torch.from_numpy(np.stack(poses)).to(dev)
    Kt = torch.from_numpy(np.stack([K_LM] * 3).astype(np.float32)).to(dev)
    dq = render_meshes(ids, P, Kt, H, W, zn, zf, quantize_bits=bits).cpu().numpy()
    d32 = render_meshes(ids, P, Kt, H, W, zn, zf).cpu().numpy()
    for i, pose in enumerate(poses):
        ref = _oracle(v, f, pose, K_LM, znear=zn, zfar=zf)
        ok = ~ref["ambiguous"] & (ref["face"] >= 0)
        assert ok.sum() > 200
        z = ref["depth"][ok]
        step = z ** 2 * (1 / zn - 1 / zf) * (2.0 ** -bits + 2.0 ** -24)
        e = (np.abs(dq[i][ok] - RO.quantize(d32[i][ok], zn, zf, bits)) / step).max()
        _note("quant", e, (bits, planes, i))
        assert e <= BARS["quant"], (bits, planes, i, e)
        e64 = np.abs(dq[i][ok] - RO.quantize(z, zn, zf, bits)) - BARS["depth"] * z - 2 * step
        assert e64.max() <= 0, (bits, planes, i)
        assert (dq[i][~ref["ambiguous"] & (ref["face"] < 0)] == 0).all()


# ------------------------------------------------------------------------------------------------ GPU: multi-mesh launches
@pytest.mark.gpu
def test_multi_mesh_launch_matches_per_roi_and_permuted(dev):
    import torch

    from gdrnpp_bop2022_b200 import _lib
    from gdrnpp_bop2022_b200.renderer import render_meshes

    meshes = [_model(dev, k, *MESHES[k]()) for k in ("ico4", "pyramid", "slivers")]
    count = _lib.lib().rast_mesh_count()
    rs = np.random.RandomState(4)
    n, h, w = 40, 120, 160
    K = K_LM.copy()
    K[:2] *= 0.25
    ids = np.array([meshes[i % 3].mesh_id for i in range(n)], np.int32)
    ids[[3, 17]] = -1
    ids[[8, 29]] = count
    ids[35] = count + 7
    poses = np.stack([_pose(_rot(100 + i), _at_pixel(K, rs.uniform(0, w), rs.uniform(0, h), rs.uniform(400, 2000)))
                      for i in range(n)])
    Ks = np.stack([K] * n).astype(np.float32)
    idt, P, Kt = torch.from_numpy(ids).to(dev), torch.from_numpy(poses).to(dev), torch.from_numpy(Ks).to(dev)
    d, xyz = render_meshes(idt, P, Kt, h, w, ZNEAR, ZFAR, return_xyz=True)
    d, xyz = d.cpu().numpy(), xyz.cpu().numpy()
    invalid = ids < 0
    invalid |= ids >= count
    assert (d[invalid] == 0).all() and (xyz[invalid] == 0).all() and (d[~invalid] > 0).any(axis=(1, 2)).all()
    for i in range(n):
        di, xi = render_meshes(idt[i:i + 1], P[i:i + 1], Kt[i:i + 1], h, w, ZNEAR, ZFAR, return_xyz=True)
        assert np.array_equal(di.cpu().numpy()[0], d[i]) and np.array_equal(xi.cpu().numpy()[0], xyz[i]), i
    perm = rs.permutation(n)
    dp = render_meshes(idt[perm], P[perm], Kt[perm], h, w, ZNEAR, ZFAR).cpu().numpy()
    assert np.array_equal(dp, d[perm])
    dt, tri, _ = _gpu(dev, ids, poses, Ks, h, w)
    assert np.array_equal(dt, d) and (tri[invalid] < 0).all()
    for i in np.nonzero(~invalid)[0][:6]:
        mk = {m.mesh_id: k for m, k in zip(meshes, ("ico4", "pyramid", "slivers"))}[ids[i]]
        v, f = MESHES[mk]()
        _compare(d[i], tri[i], xyz[i], _oracle(v, f, poses[i], Ks[i], h, w), ("multi", int(i)), sliver=mk == "slivers")


@pytest.mark.gpu
def test_more_renders_than_grid_rows(dev):
    """70 000 1x1 renders in one launch (gridDim.y is capped at 65 535): every render is drawn, unknown ids stay 0."""
    import torch

    from gdrnpp_bop2022_b200.renderer import render_meshes

    quad = np.array([[-50, -50, 0], [50, -50, 0], [50, 50, 0], [-50, 50, 0]], np.float32)
    m = _model(dev, "quad", quad, np.array([[0, 1, 2], [0, 2, 3]], np.int32))
    n = 70000
    z = 500.0 + 0.01 * np.arange(n)
    poses = np.zeros((n, 3, 4), np.float32)
    poses[:, 0, 0] = poses[:, 1, 1] = poses[:, 2, 2] = 1.0
    poses[:, 2, 3] = z
    ids = np.full(n, m.mesh_id, np.int32)
    ids[::7] = -1
    K = np.array([[500.0, 0, 0.5], [0, 500.0, 0.5], [0, 0, 1]], np.float32)
    d = render_meshes(torch.from_numpy(ids).to(dev), torch.from_numpy(poses).to(dev), torch.from_numpy(K)[None].to(dev), 1, 1,
                      ZNEAR, ZFAR).cpu().numpy()[:, 0, 0]
    assert (d[ids < 0] == 0).all()
    drawn = ids >= 0
    assert (np.abs(d[drawn] - z[drawn].astype(np.float32)) <= 5e-7 * z[drawn]).all()   # a few f32 ulps


# ------------------------------------------------------------------------------------------------ GPU: colour
@pytest.mark.gpu
@pytest.mark.parametrize("source", ("uniform", "vertex", "grey"))
def test_rgb_flat_shade_vs_oracle_faces(dev, source):
    import torch

    from gdrnpp_bop2022_b200.renderer import render_meshes_rgb

    v, f = MESHES["ico4"]()
    vc = np.random.RandomState(2).uniform(0, 1, v.shape).astype(np.float32)
    m = _model(dev, "ico4_vc", v, f, colors=vc) if source == "vertex" else _model(dev, "ico4", v, f)
    poses = [_pose(_rot(40 + i), _at_pixel(K, 320.0, 240.0, z)) for i, (K, z) in enumerate(((K_LM, 500.0), (K_SKEW, 900.0)))]
    Ks = [K_LM, K_SKEW]
    cols = np.array([[0.9, 0.4, 0.2], [0.3, 0.8, 1.0]], np.float32) if source == "uniform" else None
    rgb, _, tri = render_meshes_rgb(torch.full((2,), m.mesh_id, dtype=torch.int32, device=dev),
                                    torch.from_numpy(np.stack(poses)).to(dev),
                                    torch.from_numpy(np.stack(Ks).astype(np.float32)).to(dev), H, W, ZNEAR, ZFAR,
                                    colors=None if cols is None else torch.from_numpy(cols), return_tri_ids=True)
    rgb, tri = rgb.cpu().numpy(), tri.cpu().numpy()
    for i in range(2):
        ref = _oracle(v, f, poses[i], Ks[i])
        ok = ~ref["ambiguous"]
        assert np.array_equal(tri[i][ok], ref["face"][ok])
        exp = flat_shade(v, f, poses[i], Ks[i].astype(np.float32), ref["face"], color=None if cols is None else cols[i],
                         vert_colors=vc if source == "vertex" else None)
        e = np.abs(rgb[i].astype(np.float64) - exp)[ok].max()   # exp is unrounded: a correct rint is within 0.5
        _note("rgb", e, (source, i))
        assert e <= BARS["rgb"], (source, i, e)
        assert (rgb[i][ok & (ref["face"] < 0)] == 0).all()


# ------------------------------------------------------------------------------------------------ GPU: consumers
def _scene():
    """Two objects in mutual occlusion in one LM image: -> meshes {obj: (v, f)}, R [2,3,3], t [2,3] (mm)."""
    meshes = {1: MESHES["ico4"](), 2: _ellipsoid(4, (160.0, 60.0, 120.0))}
    R = np.stack([_rot(51), _rot(52)])
    t = np.stack([_at_pixel(K_LM, 300.0, 240.0, 800.0), _at_pixel(K_LM, 350.0, 250.0, 850.0)])
    return meshes, R, t


@pytest.mark.gpu
def test_vsd_through_gpu_renders_vs_f64_renders(dev):
    import torch

    from gdrnpp_bop2022_b200 import bop_eval
    from test_bop_eval import BOP19_TAUS, vsd_np

    meshes, R, t = _scene()
    vm = bop_eval.VsdMeshes(meshes, device=dev)
    R_e = np.stack([R[0] @ _axang(0.05, 0), R[1] @ _axang(0.08, 1)])
    t_e = t + np.array([[4.0, -3.0, 12.0], [-6.0, 2.0, -9.0]])
    gt = vm.render([1, 2], R, t, np.stack([K_LM] * 2), H, W)
    est = vm.render([1, 2], R_e, t_e, np.stack([K_LM] * 2), H, W)
    gt64 = [_oracle(*meshes[o], _pose(R[i], t[i]), K_LM, znear=bop_eval.VSD_ZNEAR, zfar=bop_eval.VSD_ZFAR)
            for i, o in enumerate((1, 2))]
    est64 = [_oracle(*meshes[o], _pose(R_e[i], t_e[i]), K_LM, znear=bop_eval.VSD_ZNEAR, zfar=bop_eval.VSD_ZFAR)
             for i, o in enumerate((1, 2))]
    both = [g["depth"] for g in gt64]
    test64 = np.where((both[0] > 0) & ((both[1] == 0) | (both[0] < both[1])), both[0], both[1]).astype(np.float32)
    amb_test = gt64[0]["ambiguous"] | gt64[1]["ambiguous"]
    g_np = gt.cpu().numpy()
    test32 = np.where((g_np[0] > 0) & ((g_np[1] == 0) | (g_np[0] < g_np[1])), g_np[0], g_np[1]).astype(np.float32)
    errs = bop_eval.vsd(est, gt, torch.from_numpy(test32[None]).to(dev), [0, 1], [0, 1], [0, 0], K_LM.astype(np.float32),
                        [120.0, 160.0], BOP19_TAUS, 15.0).cpu().numpy()
    for i in range(2):
        ref = vsd_np(est64[i]["depth"].astype(np.float32), gt64[i]["depth"].astype(np.float32), test64, K_LM.astype(np.float32),
                     15.0, BOP19_TAUS, True, (120.0, 160.0)[i])
        union = (est64[i]["depth"] > 0) | (gt64[i]["depth"] > 0)
        amb = (est64[i]["ambiguous"] | gt64[i]["ambiguous"] | amb_test) & union
        share = amb.sum() / union.sum()
        assert 0.1 < max(ref) and min(ref) < 1.0
        assert np.abs(errs[i] - np.asarray(ref)).max() <= share + 1e-12, (i, errs[i], ref, share)


def _axang(angle, axis):
    a = np.zeros(3); a[axis] = 1.0
    from oracle import gdrn_model_oracle as O

    return O.axangle2mat(a, angle)


@pytest.mark.gpu
def test_gt_info_vs_f64_renders(dev):
    from gdrnpp_bop2022_b200 import bop_eval, gt_info

    meshes, R, t = _scene()
    vm = bop_eval.VsdMeshes(meshes, device=dev)
    rs = np.random.RandomState(8)
    g0 = [_oracle(*meshes[o], _pose(R[i], t[i]), K_LM, znear=bop_eval.VSD_ZNEAR, zfar=bop_eval.VSD_ZFAR)
          for i, o in enumerate((1, 2))]
    sensor = np.where((g0[0]["depth"] > 0) & ((g0[1]["depth"] == 0) | (g0[0]["depth"] < g0[1]["depth"])), g0[0]["depth"],
                      g0[1]["depth"])
    sensor = np.round(sensor + rs.uniform(-3, 3, sensor.shape) * (sensor > 0)).astype(np.uint16)
    sensor[200:230, 300:340] = 0          # a hole in the sensor depth
    res = gt_info.annotate(vm, [1, 2], R, t, [0, 0], K_LM[None], sensor[None], [1.0], masks=True)
    Kl = K_LM.copy()
    Kl[0, 2] += W
    Kl[1, 2] += H
    for i, o in enumerate((1, 2)):
        large = _oracle(*meshes[o], _pose(R[i], t[i]), Kl, 3 * H, 3 * W, bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR)
        small = g0[i]
        info, mask, mask_visib = gt_info.host_annotation(large["depth"].astype(np.float32), small["depth"].astype(np.float32),
                                                         sensor.astype(np.float32), K_LM, 15.0)
        n_amb = int(large["ambiguous"].sum())
        ok = ~small["ambiguous"]
        assert np.array_equal(res["mask"][i][ok], mask[ok]) and np.array_equal(res["mask_visib"][i][ok], mask_visib[ok]), i
        for k in ("px_count_all", "px_count_valid", "px_count_visib"):
            assert abs(int(res[k][i]) - info[k]) <= n_amb, (i, k, int(res[k][i]), info[k], n_amb)
        assert abs(res["visib_fract"][i] - info["visib_fract"]) <= 2 * n_amb / info["px_count_all"], i
        assert info["visib_fract"] > 0.05


@pytest.mark.gpu
def test_depth_refine_in_mm_at_bop_crop(dev):
    """The batched depth refine with models in mm and a 64 x 64 crop of a YCB-V image (K scaled by 64 / 160) against the
    reference's refine arithmetic on the numpy renderer: within 1 mm (the 1e-3 m bar)."""
    import torch

    from gdrnpp_bop2022_b200.renderer import depth_refine, render_depth

    n = 4
    v, f = MESHES["ico4"]()
    model = _model(dev, "ico4", v, f)
    rs = np.random.RandomState(12)
    Ks, poses = [], []
    for i in range(n):
        z = rs.uniform(600, 1600)
        cx, cy = rs.uniform(200, 440), rs.uniform(150, 330)
        s = 64.0 / (160.0 * 900.0 / z)
        Kc = K_YCBV.copy()
        Kc[0, 2] -= cx - 80.0 * 900.0 / z
        Kc[1, 2] -= cy - 80.0 * 900.0 / z
        Kc[:2] *= s
        Ks.append(Kc.astype(np.float32))
        poses.append(_pose(_rot(70 + i), _at_pixel(K_YCBV, cx, cy, z)))
    Ks, poses = np.stack(Ks), np.stack(poses)
    true = poses.copy()
    true[:, :, 3] *= 1 + rs.uniform(-0.03, 0.03, (n, 1))
    sensor = render_depth(model, torch.from_numpy(true).to(dev), torch.from_numpy(Ks).to(dev), 64, 64, ZNEAR, ZFAR)
    xyz = (torch.rand(n, 3, 64, 64, generator=torch.Generator().manual_seed(0)) - 0.5).to(dev) * 100.0
    mask = torch.rand(n, 1, 64, 64, generator=torch.Generator().manual_seed(1)).to(dev)
    new_t = depth_refine(model, torch.from_numpy(poses[:, :, :3]).to(dev).contiguous(),
                         torch.from_numpy(poses[:, :, 3]).to(dev).contiguous(), torch.from_numpy(Ks).to(dev), xyz, mask,
                         sensor, iters=2, thresh=0.8, znear=ZNEAR, zfar=ZFAR).cpu().numpy()
    mx = mask.view(n, -1).max(1)[0].view(n, 1, 1, 1)
    mn = mask.view(n, -1).min(1)[0].view(n, 1, 1, 1)
    mnorm = ((mask - mn) / (mx - mn)).cpu().numpy()
    sens = sensor.cpu().numpy()
    for i in range(n):
        t = poses[i, :, 3].astype(np.float64).copy()
        for _ in range(2):
            ren = OO.render_depth(v, f, _pose(poses[i, :, :3], t), Ks[i], 64, 64, ZNEAR, ZFAR)
            t = OO.depth_refine_step(xyz[i].permute(1, 2, 0).cpu().numpy(), mnorm[i, 0], sens[i], ren, Ks[i], t)
        e = np.abs(new_t[i] - t).max()
        _note("refine_t", e, i)
        assert e <= BARS["refine_t"], (i, e)
        assert abs(new_t[i, 2] - true[i, 2, 3]) < abs(poses[i, 2, 3] - true[i, 2, 3])
