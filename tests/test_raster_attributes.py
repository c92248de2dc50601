"""The scene render (csrc/raster.cu: rast_render_scene, rast_upload_mesh_tex; renderer.render_scene, EGLRenderer.render)
against oracle/raster_attr_oracle.py, an f64 NumPy restatement of shader_textureless_texture.{vs,frag}, the
perspective-correct interpolation, the mip chain and the LOD rule.

The CPU tests pin the oracle to hand-worked cases (a texel-aligned quad, a known minification, the normals of a sphere,
pc_obj = R^-1 (pc_cam - t)), the PLY reader's texture fields, the EGL loader's normal and texture conventions, and the
arguments EGLRenderer.render refuses.  The GPU tests compare every output with the oracle on a 640 x 480 scene of five
mutually occluding instances of BOP-scale meshes (20 k - 30 k triangles), and pc_cam, seg and depth bit for bit with the
per-instance composite EGLRenderer.render ran before the scene render existed.

Bars (BARS) are at most 4x the largest error measured on an H100 (80GB HBM3, 700 W power limit); the measured maxima
are printed at the end of the module.
"""
import numpy as np
import pytest

from oracle import raster_attr_oracle as RA

# quantity -> bar on unambiguous covered pixels
BARS = {
    "depth": 5e-6,       # 1.34e-6  relative |z - z64| / z64
    "pc_obj": 2e-5,      # 7.33e-6  |pc_obj - pc_obj64| / 0.12 m, the ellipsoid's extent
    "normal": 2e-5,      # 7.07e-6  |normal - normal64|, the 0.5 n + 0.5 encoding
    "image": 0.03,       # 0.00795  |255 image - 255 image64|: f32 barycentrics and LOD move the sample by ~1e-7 of the
                         #          texture across 0 -> 255 texel steps; the filter weights are f32, not fixed point
}
MEASURED = {}


def _note(what, value):
    MEASURED[what] = max(MEASURED.get(what, 0.0), float(value))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(MEASURED.items()):
        print(f"measured {k}: {v:.3g}")


# ------------------------------------------------------------------------------------------------ meshes and textures
def _checker(n=256, cells=16):
    i = (np.arange(n) // (n // cells))
    c = ((i[:, None] + i[None, :]) % 2).astype(np.float64)
    tex = np.stack([40 + 200 * c, 255 - 180 * c, 90 + 60 * c], -1)
    return tex.astype(np.uint8)


def _gradient(h=192, w=320):
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([255 * x / (w - 1), 255 * y / (h - 1), 128 + 100 * np.sin(x / 9.0) * np.cos(y / 7.0)],
                    -1).round().clip(0, 255).astype(np.uint8)


def _uv_ellipsoid(subdiv=5, extent=(0.12, 0.08, 0.1)):
    """Icosphere (20480 faces at subdiv 5) scaled to an ellipsoid, spherical UVs, the unit-sphere normals."""
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    v, f = make_icosphere_mesh(subdiv, extent)
    v = np.asarray(v, np.float32)
    d = v / (np.asarray(extent, np.float32) / 2)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    uv = np.stack([0.5 + np.arctan2(d[:, 1], d[:, 0]) / (2 * np.pi), np.arccos(np.clip(d[:, 2], -1, 1)) / np.pi], 1)
    nrm = d / (np.asarray(extent) / 2)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return v, np.asarray(f, np.int32), nrm.astype(np.float32), uv.astype(np.float32)


def _grid_cube(n=40, size=0.09):
    """A cube of 6 x 2 n^2 triangles (19200 at n = 40), one vertex grid per side with its own UVs and normal."""
    vs, fs, ns, uvs = [], [], [], []
    g = np.linspace(-0.5, 0.5, n + 1)
    a, b = np.meshgrid(g, g, indexing="xy")
    for ax in range(3):
        for sgn in (-1.0, 1.0):
            p = np.zeros((n + 1, n + 1, 3))
            p[..., ax] = 0.5 * sgn
            p[..., (ax + 1) % 3] = a
            p[..., (ax + 2) % 3] = b
            base = sum(len(x) for x in vs)
            vs.append(p.reshape(-1, 3) * size)
            nn = np.zeros(3); nn[ax] = sgn
            ns.append(np.tile(nn, ((n + 1) ** 2, 1)))
            uvs.append(np.stack([a + 0.5, b + 0.5], -1).reshape(-1, 2))
            idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1) + base
            q = np.stack([idx[:-1, :-1], idx[:-1, 1:], idx[1:, 1:], idx[1:, :-1]], -1).reshape(-1, 4)
            fs.append(np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]]))
    return (np.concatenate(vs).astype(np.float32), np.concatenate(fs).astype(np.int32),
            np.concatenate(ns).astype(np.float32), np.concatenate(uvs).astype(np.float32))


def _rot(seed):
    q, r = np.linalg.qr(np.random.RandomState(seed).randn(3, 3))
    q *= np.sign(np.diag(r))
    return q * np.linalg.det(q)


K_YCBV = np.array([[1066.778, 0.0, 312.9869], [0.0, 1067.487, 241.3109], [0.0, 0.0, 1.0]])


# ------------------------------------------------------------------------------------------------ CPU: the oracle
def _quad(extent_px, f=100.0, uv_range=1.0, z=1.0):
    """A screen-aligned square covering pixels [0, extent_px) at depth z (K = diag(f, f, 1)), UVs 0..uv_range."""
    e = extent_px / f * z
    v = np.array([[0, 0, z], [e, 0, z], [e, e, z], [0, e, z]], np.float64)
    uv = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], np.float64) * uv_range
    return dict(verts=v, faces=np.array([[0, 1, 2], [0, 2, 3]]), normals=np.tile([0.0, 0.0, -1.0], (4, 1)), uvs=uv)


def _quad_render(m, tex, n_px):
    m = dict(m, texture=tex)
    K = np.array([[100.0, 0, 0], [0, 100.0, 0], [0, 0, 1]])
    P = np.hstack([np.eye(3), np.zeros((3, 1))])
    return RA.render_scene([m], [P], K, n_px + 4, n_px + 4, 0.1, 10.0, mat_diffuse=(0, 0, 0), mat_ambient=(1, 1, 1))


def test_oracle_texel_aligned_quad_returns_texels():
    tex = np.random.RandomState(0).randint(0, 256, (8, 8, 3)).astype(np.uint8)
    o = _quad_render(_quad(8), tex, 8)
    inner = ~o["ambiguous"][:8, :8]
    assert inner.sum() > 40
    assert np.abs(o["lod"][:8, :8][inner]).max() < 1e-9
    assert np.abs(o["image"][:8, :8][inner] - tex[:8, :8][inner] / 255.0).max() < 1e-9


def test_oracle_mip_chain_and_minification():
    assert RA.mip_chain(np.array([[[0] * 3, [1] * 3], [[2] * 3, [4] * 3]], np.uint8))[1][0, 0, 0] == 2   # (7 + 2) >> 2
    ch = RA.mip_chain(np.zeros((5, 3, 3), np.uint8))
    assert [c.shape[:2] for c in ch] == [(5, 3), (2, 1), (1, 1)]
    tex = np.random.RandomState(1).randint(0, 256, (32, 32, 3)).astype(np.uint8)
    chain = RA.mip_chain(tex)
    # 32 texels over 8 pixels: rho = 4, lambda = 2 -> level 2 (8 x 8) alone, one texel per pixel
    o = _quad_render(_quad(8), tex, 8)
    inner = ~o["ambiguous"][:8, :8]
    assert np.abs(o["lod"][:8, :8][inner] - 2.0).max() < 1e-9
    assert np.abs(o["image"][:8, :8][inner] - chain[2][inner] / 255.0).max() < 1e-9
    # UVs over 2^1.5 / 4 of the texture: rho = 2^1.5, lambda = 1.5 -> levels 1 and 2 half and half
    rng = 2 ** 1.5 / 4
    o = _quad_render(_quad(8, uv_range=rng), tex, 8)
    rr, cc = np.nonzero(~o["ambiguous"][:8, :8])
    s, t = (cc + 0.5) / 8 * rng, (rr + 0.5) / 8 * rng
    want = 0.5 * RA.bilinear(chain[1], s, t) + 0.5 * RA.bilinear(chain[2], s, t)
    assert np.abs(o["lod"][rr, cc] - 1.5).max() < 1e-9
    assert np.abs(o["image"][rr, cc] - want).max() < 1e-9
    # magnification (lambda < 0) is bilinear on level 0, clamped at the edges
    assert np.allclose(RA.sample(chain, np.array([-1.0]), np.array([2.0]), np.array([-3.0]))[0], tex[31, 0] / 255.0)


def test_oracle_sphere_normals_and_pc_obj():
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    v, f = make_icosphere_mesh(4, (0.2, 0.2, 0.2))
    v = np.asarray(v, np.float64)
    R, t = _rot(3), np.array([0.02, -0.01, 0.7])
    P = np.hstack([R, t[:, None]])
    m = dict(verts=v, faces=f, normals=v / np.linalg.norm(v, axis=1, keepdims=True))
    o = RA.render_scene([m], [P], K_YCBV, 240, 320, 0.1, 10.0)
    cov = (o["seg"] > 0) & ~o["ambiguous"]
    assert cov.sum() > 10000
    analytic = (o["pc_cam"][cov] - t) / np.linalg.norm(o["pc_cam"][cov] - t, axis=1, keepdims=True)
    n = 2 * o["normal"][cov] - 1
    assert np.abs(n - analytic).max() < 3e-3            # interpolated, not renormalised: the facets' chord deficit
    assert np.abs((o["pc_cam"][cov] - t) @ R - o["pc_obj"][cov]).max() < 1e-9
    assert (o["normal"][~(o["seg"] > 0)] == 0).all() and (o["image"][~(o["seg"] > 0)] == 0).all()


def test_oracle_textureless_shading_by_hand():
    """One triangle facing the camera head-on, light at the eye: diff = 1 at the centre ray, so colour (1 + 0.2)."""
    m = dict(verts=np.array([[-1, -1, 2.0], [1, -1, 2.0], [0, 1, 2.0]]), faces=np.array([[0, 1, 2]]),
             normals=np.tile([0.0, 0.0, -1.0], (3, 1)), colors=np.tile([0.5, 0.25, 0.9], (3, 1)))
    K = np.array([[10.0, 0, 5.0], [0, 10.0, 5.0], [0, 0, 1]])
    o = RA.render_scene([m], [np.hstack([np.eye(3), np.zeros((3, 1))])], K, 10, 10, 0.1, 10.0)
    L = -np.array([0.5 / 10 * 2, 0.5 / 10 * 2, 2.0])       # pixel (5, 5): ray (0.05, 0.05, 1) at z = 2
    diff = (-L[2]) / np.linalg.norm(L)
    assert np.allclose(o["image"][5, 5], np.minimum(np.array([0.5, 0.25, 0.9]) * (diff + 0.2), 1.0))
    assert np.allclose(o["normal"][5, 5], [0.5, 0.5, 0.0])


# ------------------------------------------------------------------------------------------------ CPU: loading
_PLY_HDR = """ply
format {fmt} 1.0
comment TextureFile obj_000001.png
element vertex 4
property float x
property float y
property float z
property float nx
property float ny
property float nz
property float {u}
property float {v}
element face 2
property list uchar int vertex_indices
end_header
"""
_VERTS = np.array([[0, 0, 0, 0, 0, 1, 0.0, 0.0], [1, 0, 0, 0, 0, 1, 1.0, 0.0], [1, 1, 0, 0, 0, 1, 1.0, 1.0],
                   [0, 1, 0, 0, 0, 1, 0.0, 1.0]], np.float32)
_FACES = np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def _write_textured_ply(path, binary, u="texture_u", v="texture_v"):
    with open(path, "wb") as fh:
        fh.write(_PLY_HDR.format(fmt="binary_little_endian" if binary else "ascii", u=u, v=v).encode())
        if binary:
            fh.write(_VERTS.astype("<f4").tobytes())
            rec = np.zeros(2, dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
            rec["n"], rec["i"] = 3, _FACES
            fh.write(rec.tobytes())
        else:
            for r in _VERTS:
                fh.write((" ".join("%g" % x for x in r) + "\n").encode())
            for r in _FACES:
                fh.write(("3 %d %d %d\n" % tuple(r)).encode())


@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("names", [("texture_u", "texture_v"), ("s", "t")])
def test_ply_reads_uvs_normals_and_texture_file(tmp_path, binary, names):
    from gdrnpp_bop2022_b200.ply import load_ply

    p = str(tmp_path / "m.ply")
    _write_textured_ply(p, binary, *names)
    m = load_ply(p, vertex_scale=2.0)
    assert m["texture_file"] == "obj_000001.png"
    np.testing.assert_array_equal(m["texture_uv"], _VERTS[:, 6:8])
    np.testing.assert_array_equal(m["normals"], _VERTS[:, 3:6])
    np.testing.assert_array_equal(m["pts"], _VERTS[:, :3] * 2.0)
    np.testing.assert_array_equal(m["faces"], _FACES)


def test_ply_rejects_per_face_uvs(tmp_path):
    from gdrnpp_bop2022_b200.ply import load_ply

    p = tmp_path / "faceuv.ply"
    p.write_text("ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\n"
                 "element face 1\nproperty list uchar int vertex_indices\nproperty list uchar float texcoord\n"
                 "end_header\n0 0 0\n1 0 0\n0 1 0\n3 0 1 2 6 0 0 1 0 0 1\n")
    with pytest.raises(ValueError, match="faceuv.ply.*per-face texture"):
        load_ply(str(p))


def test_calc_normals_follows_the_egl_loader():
    """meshutil.py:calc_normals: consecutive vertex triples, not faces; degenerate -> 0; a leftover vertex -> 0."""
    from gdrnpp_bop2022_b200.renderer import calc_normals

    v = np.array([[0, 0, 0], [2, 0, 0], [0, 3, 0], [1, 1, 1], [1, 1, 1], [2, 2, 2], [5, 5, 5]], np.float32)
    n = calc_normals(v)
    np.testing.assert_array_equal(n[:3], np.tile([0, 0, 1], (3, 1)))
    np.testing.assert_array_equal(n[3:], 0)


def test_load_texture_flips_and_converts(tmp_path):
    from PIL import Image

    from gdrnpp_bop2022_b200.renderer import load_texture

    im = np.random.RandomState(2).randint(0, 256, (5, 7, 3)).astype(np.uint8)
    Image.fromarray(im).save(tmp_path / "t.png")
    np.testing.assert_array_equal(load_texture(str(tmp_path / "t.png")), im[::-1])
    Image.fromarray(im[..., 0]).save(tmp_path / "g.png")
    np.testing.assert_array_equal(load_texture(str(tmp_path / "g.png")), np.repeat(im[::-1, :, :1], 3, axis=2))


@pytest.mark.parametrize("kw", [dict(instance_colors=[(1, 0, 0)]), dict(extents=[(1, 1, 1)]),
                                dict(gt_extents=[(1, 1, 1)]), dict(background=np.zeros((4, 4, 3))),
                                dict(rot_type="quat")])
def test_egl_render_refuses_unsupported_arguments(kw):
    from gdrnpp_bop2022_b200.renderer import EGLRenderer

    egl = EGLRenderer([], K=np.eye(3), width=4, height=4, device="cpu")
    with pytest.raises(NotImplementedError, match=next(iter(kw)) if "rot_type" not in kw else "rot_type"):
        egl.render([0], [np.eye(4)[:3]], **kw)


def test_egl_renderer_refuses_materialed_models():
    from gdrnpp_bop2022_b200.renderer import EGLRenderer

    with pytest.raises(NotImplementedError, match="materialed"):
        EGLRenderer(["robot.dae"], device="cpu")


# ------------------------------------------------------------------------------------------------ GPU
def _scene_meshes():
    """Five instances: a checkerboard ellipsoid, a gradient cube, a vertex-coloured ellipsoid, a cube without
    colours (the CAD grey) and the checkerboard ellipsoid again, placed to occlude one another 0.5 - 0.8 m away."""
    ev, ef, en, euv = _uv_ellipsoid()
    cv, cf, cn, cuv = _grid_cube()
    col = (0.5 + 0.5 * np.sin(ev * np.array([40.0, 55.0, 70.0]))).astype(np.float32)
    ell_tex = dict(verts=ev, faces=ef, normals=en, uvs=euv, texture=_checker())
    cube_tex = dict(verts=cv, faces=cf, normals=cn, uvs=cuv, texture=_gradient())
    ell_col = dict(verts=ev, faces=ef, normals=en, colors=col)
    cube_cad = dict(verts=cv, faces=cf, normals=cn)
    meshes = [ell_tex, cube_tex, ell_col, cube_cad, ell_tex]
    ts = [(0.0, 0.0, 0.6), (0.05, 0.03, 0.66), (-0.06, 0.02, 0.64), (0.03, -0.06, 0.7), (-0.1, -0.08, 0.8)]
    poses = [np.hstack([_rot(10 + i), np.array(t)[:, None]]).astype(np.float32) for i, t in enumerate(ts)]
    return meshes, poses


def _upload(m, dev):
    from gdrnpp_bop2022_b200.renderer import Model3D

    return Model3D(m["verts"], m["faces"], device=dev, colors=m.get("colors"), normals=m.get("normals"),
                   uvs=m.get("uvs"), texture=m.get("texture"))


@pytest.mark.gpu
def test_scene_outputs_match_oracle(dev):
    import torch

    from gdrnpp_bop2022_b200.renderer import render_scene

    meshes, poses = _scene_meshes()
    models = {}
    for m in meshes:
        if id(m) not in models:
            models[id(m)] = _upload(m, dev)
    ids = torch.tensor([models[id(m)].mesh_id for m in meshes], dtype=torch.int32, device=dev)
    H, W, zn, zf = 480, 640, 0.25, 6.0
    light = (0.3, -0.2, 0.1)
    g = render_scene(ids, torch.from_numpy(np.stack(poses)).to(dev), torch.from_numpy(K_YCBV.astype(np.float32)), H, W,
                     zn, zf, light_pos=light, light_color=(1.0, 0.9, 0.8),
                     outputs=("pc_cam", "pc_obj", "normal", "image", "seg"))
    g = {k: v.cpu().numpy().astype(np.float64) for k, v in g.items()}
    o = RA.render_scene(meshes, poses, K_YCBV, H, W, zn, zf, light_pos=light, light_color=(1.0, 0.9, 0.8))
    ok = ~o["ambiguous"]
    cov = o["seg"] > 0
    assert (cov & ok).sum() > 40000 and len(np.unique(o["seg"][cov])) == 5
    np.testing.assert_array_equal(g["seg"][ok], o["seg"][ok])           # coverage and the winning instance
    np.testing.assert_array_equal(g["depth"][ok] > 0, cov[ok])
    m = ok & cov
    for k in ("depth",):
        e = np.abs(g[k][m] - o[k][m]) / o[k][m]
        _note(k, e.max()); assert e.max() <= BARS[k]
    e = np.abs(g["pc_obj"][m] - o["pc_obj"][m]).max() / 0.12
    _note("pc_obj", e); assert e <= BARS["pc_obj"]
    e = np.abs(g["normal"][m] - o["normal"][m]).max()
    _note("normal", e); assert e <= BARS["normal"]
    e = 255 * np.abs(g["image"][m] - o["image"][m])
    _note("image", e.max()); assert e.max() <= BARS["image"]
    textured = m & np.isfinite(o["lod"])
    assert textured.sum() > 10000 and np.nanmax(o["lod"]) > 1.0         # minified texels were sampled
    bg = ok & ~cov
    for k in ("pc_cam", "pc_obj", "normal", "image"):
        assert (g[k][bg] == 0).all()


def _old_egl_composite(models, obj_ids, poses, K, H, W, zn, zf, dev):
    """EGLRenderer.render as it was before the scene render: one render_depth per instance, then the composite."""
    import torch

    from gdrnpp_bop2022_b200.renderer import render_depth

    Kt = torch.from_numpy(np.asarray(K, np.float32))[None].to(dev)
    depth = torch.zeros((H, W), device=dev)
    xyz = torch.zeros((H, W, 3), device=dev)
    seg = torch.zeros((H, W), device=dev)
    for k, (oid, pose) in enumerate(zip(obj_ids, poses)):
        p = torch.as_tensor(np.asarray(pose, np.float32)[:3, :4])[None].to(dev)
        d, x = render_depth(models[oid], p, Kt, H, W, zn, zf, return_xyz=True)
        upd = (d[0] > 0) & ((depth == 0) | (d[0] < depth))
        depth = torch.where(upd, d[0], depth)
        xyz = torch.where(upd[..., None], x[0], xyz)
        seg = torch.where(upd, torch.full_like(seg, float(k + 1)), seg)
    return depth, xyz, seg


@pytest.mark.gpu
def test_egl_pc_cam_seg_depth_bit_identical_to_per_instance_composite(dev):
    import torch

    from gdrnpp_bop2022_b200.renderer import EGLRenderer

    meshes, poses = _scene_meshes()
    models = [_upload(m, dev) for m in meshes[:4]]
    obj_ids = [0, 1, 2, 3, 0, 1]
    ps = poses[:4] + [poses[0], poses[4]]      # instance 4 repeats instance 0 exactly: every one of its depths ties
    egl = EGLRenderer(models, K=K_YCBV, width=640, height=480, device=dev)
    pc = torch.zeros((480, 640, 4), device=dev)
    seg = torch.zeros((480, 640, 4), device=dev)
    depth = egl.render(obj_ids, ps, pc_cam_tensor=pc, seg_tensor=seg)
    d0, x0, s0 = _old_egl_composite(models, obj_ids, ps, K_YCBV, 480, 640, 0.25, 6.0, dev)
    assert torch.equal(depth, d0) and torch.equal(pc[..., :3], x0) and torch.equal(seg[..., 0], s0)
    assert torch.equal(pc[..., 3], (d0 > 0).float())
    assert not (seg[..., 0] == 5).any() and (seg[..., 0] == 1).any()


@pytest.mark.gpu
def test_new_mesh_fields_leave_existing_renders_unchanged(dev):
    import torch

    from gdrnpp_bop2022_b200.renderer import Model3D, depth_refine, render_meshes, render_meshes_rgb

    ev, ef, en, euv = _uv_ellipsoid(4)
    col = np.full_like(ev, 0.7)
    plain = Model3D(ev, ef, device=dev, colors=col)
    rich = Model3D(ev, ef, device=dev, colors=col, normals=en, uvs=euv, texture=_checker(64, 8))
    untextured = Model3D(ev, ef, device=dev, colors=col, normals=en, uvs=euv)
    n = 4
    poses = torch.from_numpy(np.stack([np.hstack([_rot(20 + i), [[0.01 * i], [0.0], [0.5]]]) for i in range(n)]
                                      ).astype(np.float32)).to(dev)
    K = torch.tensor([[[266.7, 0.0, 80.3], [0.0, 266.9, 63.8], [0.0, 0.0, 1.0]]], device=dev)
    a, b = (torch.full((n,), m.mesh_id, dtype=torch.int32, device=dev) for m in (plain, rich))
    da, xa = render_meshes(a, poses, K, 128, 160, return_xyz=True)
    db, xb = render_meshes(b, poses, K, 128, 160, return_xyz=True)
    assert (da > 0).sum(dim=(1, 2)).min() > 1000
    assert torch.equal(da, db) and torch.equal(xa, xb)
    # the colour render changes only where the mesh has a texture to sample, and only its colour
    c = torch.full((n,), untextured.mesh_id, dtype=torch.int32, device=dev)
    ra = render_meshes_rgb(a, poses, K, 128, 160, return_tri_ids=True)
    rc = render_meshes_rgb(c, poses, K, 128, 160, return_tri_ids=True)
    assert all(torch.equal(x, y) for x, y in zip(ra, rc))
    rb = render_meshes_rgb(b, poses, K, 128, 160, return_tri_ids=True)
    assert torch.equal(ra[1], rb[1]) and torch.equal(ra[2], rb[2]) and not torch.equal(ra[0], rb[0])
    ucol = torch.tensor([[0.2, 0.4, 0.6]] * n, device=dev)
    assert torch.equal(render_meshes_rgb(a, poses, K, 128, 160, colors=ucol)[0],
                       render_meshes_rgb(b, poses, K, 128, 160, colors=ucol)[0])
    hw = 64
    g = torch.Generator(device="cpu").manual_seed(0)
    xyz = torch.rand((n, 3, hw, hw), generator=g).to(dev)
    mask = torch.rand((n, 1, hw, hw), generator=g).to(dev)
    sensor = (0.5 + 0.01 * torch.rand((n, hw, hw), generator=g)).to(dev)
    Kc = K.expand(n, 3, 3).contiguous() * torch.tensor([0.4, 0.4, 1.0], device=dev)[None, :, None]
    ta = depth_refine(plain, poses[:, :, :3], poses[:, :, 3], Kc, xyz, mask, sensor)
    tb = depth_refine(rich, poses[:, :, :3], poses[:, :, 3], Kc, xyz, mask, sensor)
    assert torch.equal(ta, tb) and not torch.equal(ta, poses[:, :, 3])


@pytest.mark.gpu
def test_egl_renderer_fills_every_buffer_with_reference_layouts(dev, tmp_path):
    """A reference call site (texture_paths, image_tensor, pc_obj_tensor, normal_tensor) against render_scene."""
    import torch
    from PIL import Image

    from gdrnpp_bop2022_b200.renderer import EGLRenderer, render_scene

    cv, cf, cn, cuv = _grid_cube(8)
    ply = tmp_path / "obj_000001.ply"
    hdr = ("ply\nformat binary_little_endian 1.0\ncomment TextureFile obj_000001.png\nelement vertex %d\n"
           "property float x\nproperty float y\nproperty float z\nproperty float nx\nproperty float ny\n"
           "property float nz\nproperty float texture_u\nproperty float texture_v\nelement face %d\n"
           "property list uchar int vertex_indices\nend_header\n" % (len(cv), len(cf)))
    rec = np.zeros(len(cf), dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    rec["n"], rec["i"] = 3, cf
    with open(ply, "wb") as fh:
        fh.write(hdr.encode())
        fh.write(np.hstack([cv * 1000.0, cn, cuv]).astype("<f4").tobytes())
        fh.write(rec.tobytes())
    tex = _gradient(64, 96)
    Image.fromarray(tex).save(tmp_path / "obj_000001.png")
    H, W = 120, 160
    K = np.array([[200.0, 0, 80.0], [0, 200.0, 60.0], [0, 0, 1]], np.float32)
    egl = EGLRenderer([str(ply)], K=K, width=W, height=H, vertex_scale=0.001, device=dev,
                      texture_paths=[str(tmp_path / "obj_000001.png")])
    pose = np.hstack([_rot(5), [[0.0], [0.0], [0.4]]]).astype(np.float32)
    bufs = {k: torch.full((H, W, 4), -7.0, device=dev) for k in ("image", "pc_obj", "normal", "pc_cam", "seg")}
    egl.render([0], [pose], K=K, image_tensor=bufs["image"], pc_obj_tensor=bufs["pc_obj"], normal_tensor=bufs["normal"],
               pc_cam_tensor=bufs["pc_cam"], seg_tensor=bufs["seg"], light_pos=(0.1, 0.1, 0.0))
    r = render_scene(torch.tensor([egl.models[0].mesh_id], dtype=torch.int32, device=dev),
                     torch.from_numpy(pose)[None].to(dev), torch.from_numpy(K), H, W, 0.25, 6.0,
                     light_pos=(0.1, 0.1, 0.0), outputs=("pc_obj", "normal", "image"))
    assert egl.models[0].is_textured and (r["depth"] > 0).sum() > 2000
    assert torch.equal(bufs["image"][..., :3], r["image"][..., [2, 1, 0]] * 255) and (bufs["image"][..., 3] == 255).all()
    assert torch.equal(bufs["pc_obj"][..., :3], r["pc_obj"]) and (bufs["pc_obj"][..., 3] == 1).all()
    assert torch.equal(bufs["normal"][..., :3], torch.flip(r["normal"], (0,))) and (bufs["normal"][..., 3] == 1).all()
    assert (bufs["seg"][..., 1:] == -7).all() and torch.equal(bufs["pc_cam"][..., 2], r["depth"])
    # the texture reached the image: the mean colour of a textured render is not the flat material grey
    img = r["image"][r["depth"] > 0]
    assert float(img.std(0).max()) > 0.02
    # the light persists across calls, like set_light_pos
    assert list(egl.lightpos) == [0.1, 0.1, 0.0]


# ------------------------------------------------------------------------------------------------ loaders, continued
def test_load_models_takes_the_evaluators_arguments(tmp_path, monkeypatch):
    """gdrn_evaluator.py:77-84 passes texture_paths (YCB-V sets one per object) to the depth renderer's load_models,
    which ignores it, with cache_dir / center / use_cache."""
    from gdrnpp_bop2022_b200 import renderer

    made = []
    monkeypatch.setattr(renderer, "Model3D", lambda v, f, device="cuda", **kw: made.append((v, f, kw)) or len(made))
    p = str(tmp_path / "m.ply")
    _write_textured_ply(p, True)
    ms = renderer.load_models(model_paths=[p], scale_to_meter=0.001, cache_dir=".cache",
                              texture_paths=[str(tmp_path / "obj_000001.png")], center=False, use_cache=True)
    assert ms == [1] and made[0][2] == {}
    np.testing.assert_allclose(made[0][0], _VERTS[:, :3].astype(np.float64) * 0.001, rtol=1e-7)


def test_egl_renderer_constructor_refusals_and_arguments(tmp_path, monkeypatch):
    from gdrnpp_bop2022_b200 import renderer

    for kw in (dict(model_colors=[(1, 0, 0)]), dict(render_marker=True), dict(model_loadfn="pyassimp")):
        with pytest.raises(NotImplementedError, match=next(iter(kw))):
            renderer.EGLRenderer([], device="cpu", **kw)
    made = []
    monkeypatch.setattr(renderer, "Model3D", lambda v, f, device="cuda", **kw: made.append(kw) or len(made))
    p = str(tmp_path / "grey.ply")
    from gdrnpp_bop2022_b200.ply import save_ply

    save_ply(p, _VERTS[:3, :3], _FACES[:1])
    egl = renderer.EGLRenderer([p, p], model_ids=[5, 9], cad_model_colors=[(255, 0, 51), (0, 0, 0)], device="cpu")
    assert egl.models == {5: 1, 9: 2}
    np.testing.assert_allclose(made[0]["colors"], np.tile([1.0, 0.0, 0.2], (3, 1)), rtol=1e-6)
    np.testing.assert_array_equal(made[0]["normals"], np.tile([0, 0, 1], (3, 1)))
    with pytest.raises(ValueError, match="2 obj_ids but 1 poses"):
        egl.render([5, 9], [np.eye(4)[:3]], K=np.eye(3))


# ------------------------------------------------------------------------------------------------ GPU: renderer_py texture
def _nearest_shade(verts, faces, uvs, tex, pose, K, tri):
    """render_meshes_rgb's textured flat shade restated in f64: light_w (flat_shade_oracle) times the nearest level-0
    texel at the perspective-correct UV, clamp to edge -> ([H,W,3] in [0,255], [H,W] bool: UV within 1e-4 texel of a
    texel boundary, where f32 may pick the neighbour)."""
    from oracle.flat_shade_oracle import flat_shade

    lw = flat_shade(verts, faces, pose, K, tri, color=(1.0, 1.0, 1.0))[..., :1] / 255.0
    H, W = tri.shape
    rr, cc = np.nonzero(tri >= 0)
    f = np.asarray(faces)[tri[rr, cc]]
    P = np.asarray(verts, np.float64) @ np.asarray(pose, np.float64)[:, :3].T + np.asarray(pose, np.float64)[:, 3]
    Pk = P[f]
    u = (K[0, 0] * Pk[..., 0] + K[0, 1] * Pk[..., 1]) / Pk[..., 2] + K[0, 2]
    v = K[1, 1] * Pk[..., 1] / Pk[..., 2] + K[1, 2]
    sx, sy = cc + 0.5, rr + 0.5
    A = (u[:, 1] - u[:, 0]) * (v[:, 2] - v[:, 0]) - (u[:, 2] - u[:, 0]) * (v[:, 1] - v[:, 0])
    w0 = ((u[:, 1] - sx) * (v[:, 2] - sy) - (u[:, 2] - sx) * (v[:, 1] - sy)) / A
    w1 = ((u[:, 2] - sx) * (v[:, 0] - sy) - (u[:, 0] - sx) * (v[:, 2] - sy)) / A
    w = np.stack([w0, w1, 1 - w0 - w1], 1) / Pk[..., 2]
    b = w / w.sum(1, keepdims=True)
    st = np.einsum("mk,mkc->mc", b, np.asarray(uvs, np.float64)[f])
    h, wt = tex.shape[:2]
    x, y = st[:, 0] * wt, st[:, 1] * h
    near = (np.abs(x - np.rint(x)) < 1e-4) | (np.abs(y - np.rint(y)) < 1e-4)
    i = np.clip(np.floor(x), 0, wt - 1).astype(np.int64)
    j = np.clip(np.floor(y), 0, h - 1).astype(np.int64)
    out = np.zeros((H, W, 3))
    out[rr, cc] = tex[j, i].astype(np.float64)
    amb = np.zeros((H, W), bool)
    amb[rr, cc] = near
    return lw * out, amb


@pytest.mark.gpu
def test_render_meshes_rgb_textured_matches_restatement(dev):
    import torch

    from gdrnpp_bop2022_b200.renderer import Model3D, render_meshes_rgb

    cv, cf, cn, cuv = _grid_cube(30)
    tex = _gradient(96, 160)
    m = Model3D(cv * 1000.0, cf, device=dev, uvs=cuv, texture=tex)
    n = 3
    poses = np.stack([np.hstack([_rot(30 + i), [[20.0 * i - 20], [10.0], [500.0 + 50 * i]]]) for i in range(n)])
    K = K_YCBV.astype(np.float32)
    rgb, depth, tri = render_meshes_rgb(torch.full((n,), m.mesh_id, dtype=torch.int32, device=dev),
                                        torch.from_numpy(poses.astype(np.float32)).to(dev),
                                        torch.from_numpy(K)[None].to(dev), 240, 320, 10.0, 10000.0, return_tri_ids=True)
    rgb, tri = rgb.cpu().numpy().astype(np.float64), tri.cpu().numpy()
    worst = 0.0
    for i in range(n):
        exp, amb = _nearest_shade(cv * 1000.0, cf, cuv, tex, poses[i].astype(np.float32), K.astype(np.float64), tri[i])
        ok = (tri[i] >= 0) & ~amb
        assert ok.sum() > 3000
        worst = max(worst, float(np.abs(rgb[i][ok] - exp[ok]).max()))
    _note("rgb_textured", worst)
    assert worst <= 1.0          # u8 rounding of lw * texel, as the untextured flat shade's bar


@pytest.mark.gpu
def test_vis_poses_orig_color_draws_textured_models(dev, tmp_path):
    """vis_poses --vis_orig_color on a synthetic split whose obj 1 is a textured PLY: the driver's images equal the
    in-memory composite of the library's renders, and those renders sample the texture."""
    import os

    import torch
    from PIL import Image

    from gdrnpp_bop2022_b200 import bop_eval, gt_info
    from gdrnpp_bop2022_b200 import vis_poses as VP
    from gdrnpp_bop2022_b200.ply import load_ply
    from gdrnpp_bop2022_b200.renderer import load_texture
    from gdrnpp_bop2022_b200.synthetic import write_bop_tree

    root = str(tmp_path / "datasets")
    write_bop_tree(root, dataset="ycbv", num_images=2, num_scenes=1, H=120, W=160, dets_per_image=2, obj_ids=[1, 2])
    sp = gt_info.split_params(os.path.join(root, "BOP_DATASETS"), "ycbv", "test")
    mdir = os.path.join(sp["base_path"], "models_eval")
    p = os.path.join(mdir, "obj_000001.ply")
    m = load_ply(p)
    pts = np.asarray(m["pts"], np.float64)
    span = pts.max(0) - pts.min(0)
    uv = (pts[:, :2] - pts.min(0)[:2]) / np.maximum(span[:2], 1e-9)
    hdr = ("ply\nformat binary_little_endian 1.0\ncomment TextureFile obj_000001.png\nelement vertex %d\n"
           "property float x\nproperty float y\nproperty float z\nproperty float texture_u\nproperty float texture_v\n"
           "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(pts), len(m["faces"])))
    rec = np.zeros(len(m["faces"]), dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    rec["n"], rec["i"] = 3, m["faces"]
    with open(p, "wb") as fh:
        fh.write(hdr.encode())
        fh.write(np.hstack([pts, uv]).astype("<f4").tobytes())
        fh.write(rec.tobytes())
    Image.fromarray(_checker(64, 8)).save(os.path.join(mdir, "obj_000001.png"))
    res = VP.run_split(sp, mdir, str(tmp_path / "vis"), "ycbv", "test", vis_orig_color=True, device=dev)
    assert res["images"] == 2
    # the same split in memory, with the meshes uploaded as the driver uploads them
    m1, m2 = load_ply(p), load_ply(os.path.join(mdir, "obj_000002.ply"))
    col2 = None
    if "colors" in m2:
        col2 = m2["colors"] / 255.0 if m2["colors"].max() > 1.0 else m2["colors"]
    tex = load_texture(os.path.join(mdir, "obj_000001.png"))
    meshes = bop_eval.VsdMeshes({1: (m1["pts"], m1["faces"], None, m1["texture_uv"], tex),
                                 2: (m2["pts"], m2["faces"], col2)}, device=dev)
    images = VP.plan_images(sp)
    seen_tex = False
    for scene_id, im_id, K, scale, dpath, ipath, poses in images:
        rgb = VP.read_rgb(ipath)
        depth = gt_info.read_depth(dpath).astype(np.float32) * np.float32(scale)
        o = VP.vis_object_poses(meshes, [poses], K[None], rgb[None], depth[None])[0]
        got = np.asarray(Image.open(os.path.join(str(tmp_path / "vis"), "ycbv", "test", "{:06d}".format(scene_id),
                                                 "{:06d}.jpg".format(im_id))))
        exp = np.asarray(Image.open(__import__("io").BytesIO(_jpg_bytes(o["rgb"]))))
        assert np.array_equal(got, exp)
        m_rgb, _, _ = VP.render_instances(meshes, [poses], K[None], rgb.shape[0], rgb.shape[1])
        for k, pz in enumerate(poses):
            if int(pz["obj_id"]) == 1:
                px = m_rgb[k].reshape(-1, 3)
                px = px[(px > 0).any(1)]
                seen_tex |= bool(len(px) > 50 and torch.unique(px, dim=0).shape[0] > 8)
        torch.cuda.synchronize()
    assert seen_tex


def _jpg_bytes(im):
    import io

    from PIL import Image

    buf = io.BytesIO()
    Image.fromarray(im).save(buf, format="JPEG", quality=95)
    return buf.getvalue()
