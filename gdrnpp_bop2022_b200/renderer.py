"""CUDA depth rasteriser + fast depth refinement behind the reference's renderer / evaluator surfaces.

Mirrors:
  * lib/render_vispy/renderer.py  Renderer(size, cam).{clear, set_cam, draw_model, finish} -> (rgb, depth)
    (the renderer fast depth refine uses: engine/gdrn_evaluator.py:64-84,520-526; demo/predictor_gdrn.py:100-109)
  * lib/egl_renderer/egl_renderer_v3.py  EGLRenderer(..., texture_paths=).render(obj_ids, poses, K=, image_tensor=,
    seg_tensor=, normal_tensor=, pc_obj_tensor=, pc_cam_tensor=, ...): one scene render for all instances
  * GDRN_Evaluator.process_depth_refine (engine/gdrn_evaluator.py:461-573) == GdrnPredictor.process_depth_refine
    (demo/predictor_gdrn.py:195-286), batched over ROIs on the GPU.
  * get_out_mask / get_out_coor (engine/engine_utils.py:295-333), get_K_crop_resize (core/utils/camera_geometry.py:6-21)
No GL / EGL anywhere; no CPU fallback.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib


def _f32c(t, dev=None):
    return t.detach().to(device=dev or t.device, dtype=torch.float32).contiguous()


def render_depth(model, poses, Ks, H, W, znear=0.1, zfar=100.0, quantize_bits=0, return_xyz=False):
    """One Model3D at poses [n,3,4] with Ks [n,3,3] (or one [1,3,3]) -> depth [n,H,W] (0 = background), rendered on the
    model's device: render_meshes with the model's registry id for every ROI."""
    dev = model.vertices.device
    poses = _f32c(poses, dev).reshape(-1, 3, 4)
    ids = torch.full((poses.shape[0],), model.mesh_id, dtype=torch.int32, device=dev)
    return render_meshes(ids, poses, Ks, H, W, znear, zfar, quantize_bits, return_xyz)


def get_out_mask(pred_mask, mask_loss_type="L1"):
    """engine_utils.py:313-333 (L1: per-ROI min-max normalisation to [0,1])."""
    bs = pred_mask.shape[0]
    if mask_loss_type == "L1":
        mx = torch.max(pred_mask.view(bs, -1), dim=-1)[0].view(bs, 1, 1, 1)
        mn = torch.min(pred_mask.view(bs, -1), dim=-1)[0].view(bs, 1, 1, 1)
        return (pred_mask - mn) / (mx - mn)
    if mask_loss_type in ("BCE", "RW_BCE", "dice"):
        return torch.sigmoid(pred_mask)
    raise NotImplementedError(mask_loss_type)


def get_out_coor(coor_x, coor_y, coor_z):
    """engine_utils.py:295-310 (regression branch)."""
    return torch.cat([coor_x, coor_y, coor_z], dim=1)


def get_K_crop_resize(K, crop_xy, resize_ratio):
    """core/utils/camera_geometry.py:6-21."""
    bs = K.shape[0]
    new_K = K.clone()
    new_K[:, [0, 1], 2] = K[:, [0, 1], 2] - crop_xy
    new_K[:, [0, 1]] = new_K[:, [0, 1]] * resize_ratio.view(bs, -1, 1)
    return new_K


@_lib.on_device(1)
def render_meshes(mesh_ids, poses, Ks, H, W, znear=0.1, zfar=100.0, quantize_bits=0, return_xyz=False):
    """One render per ROI of the REGISTERED mesh `mesh_ids[i]` (int32 CUDA tensor of registry ids): poses [n,3,4],
    Ks [n,3,3] -> depth [n,H,W].  The multi-object form of the reference's per-object draw loop, one launch, no sync."""
    dev = poses.device
    poses = _f32c(poses).reshape(-1, 3, 4)
    n = poses.shape[0]
    Ks = _f32c(Ks, dev).reshape(-1, 3, 3)
    if Ks.shape[0] == 1 and n > 1:
        Ks = Ks.expand(n, 3, 3).contiguous()
    ids = mesh_ids.detach().to(device=dev, dtype=torch.int32).contiguous()
    depth = torch.empty((n, H, W), dtype=torch.float32, device=dev)
    xyz = torch.empty((n, H, W, 3), dtype=torch.float32, device=dev) if return_xyz else None
    scratch = torch.empty((n * H * W,), dtype=torch.int64, device=dev)
    _lib.check(_lib.lib().rast_render_meshes(_lib.ptr(ids), _lib.ptr(poses), _lib.ptr(Ks), n, H, W, float(znear), float(zfar),
                                             int(quantize_bits), _lib.ptr(depth), _lib.ptr(xyz), _lib.ptr(scratch),
                                             _lib.current_stream()), "rast_render_meshes")
    return (depth, xyz) if return_xyz else depth


@_lib.on_device(1)
def render_meshes_rgb(mesh_ids, poses, Ks, H, W, znear=0.1, zfar=100.0, colors=None, return_tri_ids=False):
    """render_meshes in colour: the registered meshes `mesh_ids` [n] at poses [n,3,4] with Ks [n,3,3], flat-shaded as
    lib/pysixd/renderer_py.py shades them (light at the eye, ambient 0.5) -> (rgb [n,H,W,3] u8, depth [n,H,W] f32),
    plus tri_ids [n,H,W] i32 (-1 = background) with return_tri_ids.  colors [n,3] in [0,1]: a uniform colour per
    render; without it each mesh's texture (the nearest level-0 texel at the interpolated UV, clamp to edge, as
    renderer_py's texture2D), else its vertex colours, else grey 0.5.  Depth and coverage
    equal render_meshes(quantize_bits=0).  One launch set, no sync."""
    dev = poses.device
    poses = _f32c(poses).reshape(-1, 3, 4)
    n = poses.shape[0]
    Ks = _f32c(Ks, dev).reshape(-1, 3, 3)
    if Ks.shape[0] == 1 and n > 1:
        Ks = Ks.expand(n, 3, 3).contiguous()
    ids = mesh_ids.detach().to(device=dev, dtype=torch.int32).contiguous()
    cols = None if colors is None else _f32c(torch.as_tensor(colors), dev).reshape(n, 3)
    rgb = torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev)
    depth = torch.empty((n, H, W), dtype=torch.float32, device=dev)
    tri = torch.empty((n, H, W), dtype=torch.int32, device=dev) if return_tri_ids else None
    scratch = torch.empty((n * H * W,), dtype=torch.int64, device=dev)
    _lib.check(_lib.lib().rast_render_meshes_rgb(_lib.ptr(ids), _lib.ptr(poses), _lib.ptr(Ks), _lib.ptr(cols), n, H, W,
                                                 float(znear), float(zfar), _lib.ptr(rgb), _lib.ptr(depth), _lib.ptr(tri),
                                                 _lib.ptr(scratch), _lib.current_stream()), "rast_render_meshes_rgb")
    return (rgb, depth, tri) if return_tri_ids else (rgb, depth)


@_lib.on_device(1)
def depth_refine(models, rot, trans, K_crop, xyz, mask, depth_sensor, iters=2, thresh=0.8, mesh_ids=None,
                 znear=0.1, zfar=100.0, mask_loss_type="L1", coor_z_refine=False):
    """Batched fast depth refine (gdrn_evaluator.py:515-561): `iters` x (render depth at the current pose ->
    weighted-median depth offset along the weighted-centroid ray).  The weights are ||xyz|| * mask, or with
    coor_z_refine (TEST.USE_COOR_Z_REFINE, :528-537) the camera-frame z of the rotated coordinates, (rot @ xyz)_z * mask.

    models: one Model3D, or a sequence of them with `mesh_ids` [n] indexing it per ROI.
    rot [n,3,3], trans [n,3], K_crop [n,3,3], xyz [n,3,h,w] (coor maps), mask [n,1,h,w] RAW visible-mask output
    (get_out_mask -- per-ROI min-max for the L1 head, sigmoid otherwise -- runs inside the refine kernel),
    depth_sensor [n,h,w] metres.  Returns refined trans [n,3].  Per iteration: one render launch over all ROIs (every
    ROI picks its mesh from the library's registry by id) + one refine launch; no host loop over meshes, no sync."""
    dev = rot.device
    n = rot.shape[0]
    hw = xyz.shape[-1]
    rot = _f32c(rot)
    t = _f32c(trans).clone()
    K_crop = _f32c(K_crop)
    xyz = _f32c(xyz)
    raw_mask = _f32c(mask).reshape(n, hw, hw)
    if mask_loss_type == "L1":
        mask_mode = 1
    elif mask_loss_type in ("BCE", "RW_BCE", "dice"):
        mask_mode = 2
    else:
        raise NotImplementedError(mask_loss_type)
    sensor = _f32c(depth_sensor).reshape(n, hw, hw)
    L = _lib.lib()
    models = [models] if isinstance(models, Model3D) else list(models)
    reg = torch.tensor([m.mesh_id for m in models], dtype=torch.int32, device=dev)   # sequence index -> registry id
    if mesh_ids is None:
        ids = reg[:1].expand(n).contiguous()
    else:
        ids = reg[torch.as_tensor(mesh_ids).to(device=dev, dtype=torch.long)].contiguous()
    weight_mode = 1 if coor_z_refine else 0
    for _ in range(iters):
        poses = torch.cat([rot, t[:, :, None]], dim=2).contiguous()
        ren = render_meshes(ids, poses, K_crop, hw, hw, znear, zfar)
        _lib.check(L.gdrn_depth_refine_step(_lib.ptr(xyz), _lib.ptr(raw_mask), mask_mode, _lib.ptr(sensor), _lib.ptr(ren),
                                            _lib.ptr(K_crop), _lib.ptr(rot), weight_mode, _lib.ptr(t), n, hw, float(thresh),
                                            _lib.current_stream()), "gdrn_depth_refine_step")
    return t


@_lib.on_device(0)
def depth_refine_trace(xyz, mask, depth_sensor, ren, K_crop, trans, rot=None, mask_mode=1, weight_mode=0, thresh=0.8):
    """One refine step of depth_refine on a given render, with a record of every stage (gdrn_depth_refine_trace), for
    tests.  xyz [n,3,hw,hw], mask [n,hw,hw] (mask_mode 0 normalised, 1 raw L1, 2 logits), depth_sensor and ren
    [n,hw,hw], K_crop [n,3,3], trans [n,3], rot [n,3,3] (weight_mode 1 only).  Returns a dict of tensors on the device:
    t [n,3] (the refined translation, as gdrn_depth_refine_step returns it) and the trace m_lo, m_scale [n], w [n,hw,hw],
    sum [n] f64, max, min, cut [n], sel [n,hw,hw] bool, count [n], median [n], centroid [n,2] f64 (y, x), ray [n,3] f64
    and t_trace [n,3].  Entries a ROI does not reach hold NaN (count -1)."""
    if not xyz.is_cuda:
        raise _lib.GdrnError("depth_refine_trace needs CUDA tensors (no CPU fallback)")
    dev = xyz.device
    n, hw = xyz.shape[0], xyz.shape[-1]
    xyz, K_crop = _f32c(xyz), _f32c(K_crop)
    mask, sensor, ren = (_f32c(a).reshape(n, hw, hw) for a in (mask, depth_sensor, ren))
    rot = None if rot is None else _f32c(rot)
    f32 = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=dev)
    f64 = lambda *s: torch.full(s, float("nan"), dtype=torch.float64, device=dev)
    out = dict(t=_f32c(trans).clone(), m_lo=f32(n), m_scale=f32(n), w=f32(n, hw, hw), sum=f64(n), max=f32(n), min=f32(n),
               cut=f32(n), sel=torch.zeros((n, hw, hw), dtype=torch.uint8, device=dev),
               count=torch.full((n,), -1, dtype=torch.int32, device=dev), median=f32(n), centroid=f64(n, 2), ray=f64(n, 3),
               t_trace=f32(n, 3))
    P = lambda k: _lib.ptr(out[k])
    _lib.check(_lib.lib().gdrn_depth_refine_trace(_lib.ptr(xyz), _lib.ptr(mask), int(mask_mode), _lib.ptr(sensor), _lib.ptr(ren),
                                                  _lib.ptr(K_crop), _lib.ptr(rot), int(weight_mode), P("t"), n, hw, float(thresh),
                                                  P("m_lo"), P("m_scale"), P("w"), P("sum"), P("max"), P("min"), P("cut"),
                                                  P("sel"), P("count"), P("median"), P("centroid"), P("ray"), P("t_trace"),
                                                  _lib.current_stream()), "gdrn_depth_refine_trace")
    out["sel"] = out["sel"].bool()
    return out


class Model3D:
    """Minimal stand-in for lib/render_vispy/model3d.py objects: vertices [V,3] in metres + triangle indices [F,3] on
    `device`, and mesh_id, the mesh's id in the library's registry.  The mesh is uploaded once, here; the registry never
    frees, so the id stays valid for the life of the process and every render of this model goes through it.
    colors: optional per-vertex RGB [V,3] in [0,1], which render_meshes_rgb interpolates.  normals [V,3], uvs [V,2]
    and texture [h,w,3] u8 (row 0 at t = 0, the image flipped as GL takes it; needs uvs): optional shading attributes
    for EGLRenderer.render; with any of them the mesh is uploaded through rast_upload_mesh_tex."""

    def __init__(self, vertices, faces, device="cuda", colors=None, normals=None, uvs=None, texture=None):
        v = torch.as_tensor(np.ascontiguousarray(vertices, np.float32))
        f = torch.as_tensor(np.ascontiguousarray(faces, np.int32))
        c = None
        if colors is not None:
            c = torch.as_tensor(np.ascontiguousarray(colors, np.float32))
            if tuple(c.shape) != (v.shape[0], 3):
                raise _lib.GdrnError(f"Model3D: colors must be [V,3] = [{v.shape[0]},3], got {tuple(c.shape)}")
        n = uv = tex = None
        if normals is not None:
            n = torch.as_tensor(np.ascontiguousarray(normals, np.float32))
            if tuple(n.shape) != (v.shape[0], 3):
                raise _lib.GdrnError(f"Model3D: normals must be [V,3] = [{v.shape[0]},3], got {tuple(n.shape)}")
        if uvs is not None:
            uv = torch.as_tensor(np.ascontiguousarray(uvs, np.float32))
            if tuple(uv.shape) != (v.shape[0], 2):
                raise _lib.GdrnError(f"Model3D: uvs must be [V,2] = [{v.shape[0]},2], got {tuple(uv.shape)}")
        if texture is not None:
            tex = torch.as_tensor(np.ascontiguousarray(texture, np.uint8))
            if tex.ndim != 3 or tex.shape[2] != 3:
                raise _lib.GdrnError(f"Model3D: texture must be [h,w,3] u8, got {tuple(tex.shape)}")
            if uv is None:
                raise _lib.GdrnError("Model3D: a texture needs per-vertex uvs")
        with torch.cuda.device(device):   # the registry lives on the device current at the upload
            if n is None and uv is None and tex is None:
                mid = _lib.lib().rast_upload_mesh_ex(_lib.ptr(v), int(v.shape[0]), _lib.ptr(f), int(f.shape[0]), _lib.ptr(c))
            else:
                th, tw = (0, 0) if tex is None else (int(tex.shape[0]), int(tex.shape[1]))
                mid = _lib.lib().rast_upload_mesh_tex(_lib.ptr(v), int(v.shape[0]), _lib.ptr(f), int(f.shape[0]),
                                                      _lib.ptr(c), _lib.ptr(n), _lib.ptr(uv), _lib.ptr(tex), th, tw)
        if mid < 0:
            raise _lib.GdrnError(f"rast_upload_mesh failed (code {mid}): {_lib.last_error()}")
        self.mesh_id = mid
        self.vertices = v.to(device)
        self.faces = f.to(device)
        self.is_textured = tex is not None


def calc_normals(vertices):
    """The EGL loader's normals for a PLY without them (lib/egl_renderer/glutils/meshutil.py:calc_normals): the vertex
    array is read as a triangle soup, so vertices 3k, 3k+1, 3k+2 all get the unit normal of the triangle they form,
    cross(v1 - v0, v2 - v0) / |.|, or 0 when it is degenerate.  The faces are not consulted.  A trailing one or two
    vertices (V not a multiple of 3) get 0; there the reference leaves the first uninitialised and fails on the second."""
    v = np.asarray(vertices, np.float64)
    out = np.zeros_like(v)
    m = (len(v) // 3) * 3
    if m:
        t = v[:m].reshape(-1, 3, 3)
        nrm = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
        ln = np.linalg.norm(nrm, axis=1, keepdims=True)
        out[:m] = np.repeat(np.where(ln > 0, nrm / np.where(ln > 0, ln, 1.0), 0.0), 3, axis=0)
    return out.astype(np.float32)


def load_texture(path):
    """A texture image as the EGL loader hands it to GL (meshutil.py:loadTexture): decoded by PIL, converted to RGB
    when it is not (grey, palette, alpha dropped), and flipped top to bottom, so row 0 is t = 0 -> [h,w,3] u8."""
    from PIL import Image

    with Image.open(path) as im:
        rgb = np.asarray(im if im.mode == "RGB" else im.convert("RGB"), dtype=np.uint8)
    return np.ascontiguousarray(rgb[::-1])


def load_models(model_paths, scale_to_meter=1.0, device="cuda", texture_paths=None, shading=False,
                cad_model_colors=None, **_):
    """lib/render_vispy/model3d.py:load_models surface: PLY paths -> Model3D list (vertices * scale_to_meter).
    Without shading (the depth renders) texture_paths is ignored, as the vispy path's depth read-back ignores it.
    With shading (EGLRenderer) each model also carries what lib/egl_renderer/glutils/meshutil.py:load_mesh_sixd gives
    the EGL shader: the PLY's normals or calc_normals, its vertex colours (divided by 255 when any exceeds 1.1) and,
    when texture_paths[i] is a non-empty path, that texture (load_texture) with the PLY's per-vertex UVs.  A model
    with neither colours nor texture is drawn in cad_model_colors[i] (0-255 RGB, meshutil.py:483-490) when given, else
    in the CAD grey (223, 214, 205)."""
    from .ply import load_ply

    out = []
    for i, p in enumerate(model_paths):
        m = load_ply(p, vertex_scale=scale_to_meter)
        if "faces" not in m:
            raise ValueError(f"{p}: the rasteriser needs a triangle mesh (no face element)")
        if not shading:
            out.append(Model3D(m["pts"], m["faces"], device=device))
            continue
        tex_path = texture_paths[i] if texture_paths is not None else ""
        pts = np.asarray(m["pts"], np.float32)
        normals = m["normals"] if "normals" in m else calc_normals(pts)
        colors = None
        if "colors" in m:
            colors = np.asarray(m["colors"], np.float32)
            if colors.max() > 1.1:
                colors = colors / 255.0
        uvs = tex = None
        if tex_path:
            if "texture_uv" not in m:
                raise ValueError(f"{p}: texture {tex_path} given, but the PLY has no per-vertex texture_u / texture_v")
            uvs, tex = m["texture_uv"], load_texture(tex_path)
        elif colors is None and cad_model_colors is not None:
            colors = np.tile(np.asarray(cad_model_colors[i], np.float32) / 255.0, (len(pts), 1))
        out.append(Model3D(pts, m["faces"], device=device, colors=colors, normals=normals, uvs=uvs, texture=tex))
    return out


class Renderer:
    """lib/render_vispy/renderer.py:Renderer surface (:78-182): Renderer(size, cam, model_paths=, scale_to_meter=),
    set_cam / clear / draw_model / finish -> (rgb, depth).  Depth comes from the CUDA rasteriser with the vispy path's
    z-buffer read-back emulated (fixed-point window depth, decode mult / (d + addi), :176-182); rgb is not rendered
    (depth refine, the only caller on the hot path, ignores it) and is returned as zeros."""

    def __init__(self, size, cam, model_paths=None, scale_to_meter=1.0, gpu_id=None, device="cuda", depth_bits=24):
        self.width, self.height = size
        self.size = tuple(size)
        self.shape = (self.height, self.width)
        self.device = torch.device(device if gpu_id is None else "cuda:%d" % gpu_id)
        self.depth_bits = depth_bits      # GL depth attachment precision emulated by finish() (0 = float z)
        self.models = None
        if model_paths is not None:
            self.models = load_models(model_paths, scale_to_meter=scale_to_meter, device=self.device)
        self.set_cam(cam)
        self._draws = []

    def set_cam(self, cam, clip_near=0.1, clip_far=100.0):
        self.cam = np.asarray(cam, np.float32)
        self.clip_near, self.clip_far = clip_near, clip_far

    def clear(self, color=True, depth=True):
        self._draws = []

    def draw_model(self, model, pose, ambient_weight=0.5, light=(0, 0, 1), light_col=(1, 1, 1)):
        self._draws.append((model, np.asarray(pose, np.float32)[:3, :4]))

    def finish(self, only_color=False, to_255=False):
        rgb = np.zeros(self.shape + (3,), np.uint8 if to_255 else np.float32)
        if only_color:
            return rgb
        depth = None
        K = torch.from_numpy(self.cam)[None].to(self.device)
        for model, pose in self._draws:
            d = render_depth(model, torch.from_numpy(pose)[None].to(self.device), K, self.height, self.width,
                             self.clip_near, self.clip_far, quantize_bits=self.depth_bits)[0]
            if depth is None:
                depth = d
            else:  # nearest surface wins across draws (shared z-buffer in GL)
                depth = torch.where((d > 0) & ((depth == 0) | (d < depth)), d, depth)
        if depth is None:
            depth = torch.zeros(self.shape, device=self.device)
        return rgb, depth.cpu().numpy()


# Material of the EGL shader for a PLY model: lib/egl_renderer/glutils/meshutil.py:load_mesh_pyassimp takes it from the
# material pyassimp gives a PLY, whose defaults its comment at :278 records (ambient 0.05, diffuse 0.6, specular 0.6).
# The specular term never shows (see render_scene), so only diffuse and ambient are used.
EGL_MAT_DIFFUSE = (0.6, 0.6, 0.6)
EGL_MAT_AMBIENT = (0.05, 0.05, 0.05)


@_lib.on_device(1)
def render_scene(mesh_ids, poses, K, H, W, znear=0.25, zfar=6.0, light_pos=(0.0, 0.0, 0.0), light_color=(1.0, 1.0, 1.0),
                 outputs=("pc_cam", "seg"), mat_diffuse=EGL_MAT_DIFFUSE, mat_ambient=EGL_MAT_AMBIENT, background=None):
    """The registered meshes `mesh_ids` [n] (int32 CUDA) at poses [n,3,4] rendered into ONE image with one z-buffer and
    one K [3,3] (rast_render_scene): the draw loop of egl_renderer_v3.py:998-1177 in one launch set, no sync.  A depth
    tie between instances goes to the earlier one.  -> dict with depth [H,W] and each requested output of
    "pc_cam" [H,W,3] (camera-space point), "pc_obj" [H,W,3] (model-space point), "normal" [H,W,3] (0.5 n + 0.5 of the
    interpolated camera-frame normal), "image" [H,W,3] (RGB in [0,1], shader_textureless_texture.frag) and "seg" [H,W]
    (instance index + 1); every output is 0 on background and rows run top to bottom.  The light is in the camera
    frame (the EGL renderer's view matrix is the identity).  background: optional [H,W,3] u8 CUDA tensor; where no
    instance covers a pixel, "image" takes background / 255 (f32, channels as given).  It changes no other output
    (rast_render_scene_bg)."""
    dev = poses.device
    poses = _f32c(poses).reshape(-1, 3, 4)
    n = poses.shape[0]
    K = _f32c(torch.as_tensor(K), dev).reshape(3, 3)
    ids = mesh_ids.detach().to(device=dev, dtype=torch.int32).contiguous()
    unknown = set(outputs) - {"pc_cam", "pc_obj", "normal", "image", "seg"}
    if unknown:
        raise ValueError(f"render_scene: unknown outputs {sorted(unknown)}")
    if background is not None:
        if background.dtype != torch.uint8 or tuple(background.shape) != (H, W, 3) or background.device != dev:
            raise ValueError(f"render_scene: background must be a [{H},{W},3] uint8 tensor on {dev}, got "
                             f"{tuple(background.shape)} {background.dtype} on {background.device}")
        background = background.contiguous()
    out = {"depth": torch.empty((H, W), dtype=torch.float32, device=dev)}
    for k in outputs:
        out[k] = torch.empty((H, W) if k == "seg" else (H, W, 3), dtype=torch.float32, device=dev)
    if n == 0 and (background is None or "image" not in outputs):
        return {k: v.zero_() for k, v in out.items()}
    light = (ctypes.c_float * 12)(*[float(x) for x in (*light_pos, *light_color, *mat_diffuse, *mat_ambient)])
    L = _lib.lib()
    scratch = torch.empty((L.rast_scene_scratch_bytes(n, H, W) // 8,), dtype=torch.int64, device=dev)
    P = lambda k: _lib.ptr(out.get(k))
    _lib.check(L.rast_render_scene_bg(_lib.ptr(ids), _lib.ptr(poses), n, _lib.ptr(K), H, W, float(znear), float(zfar),
                                      light, _lib.ptr(background), P("depth"), P("pc_cam"), P("pc_obj"), P("normal"),
                                      P("image"), P("seg"), _lib.ptr(scratch), _lib.current_stream()),
               "rast_render_scene_bg")
    return out


class EGLRenderer:
    """lib/egl_renderer/egl_renderer_v3.py:EGLRenderer surface (:50-67, 838-857, 1183-1228):
    EGLRenderer(model_paths, K=, width=, height=, vertex_scale=, znear=, zfar=, texture_paths=) and
    render(obj_ids, poses, K=, to_bgr=, to_255=, light_pos=, light_color=, image_tensor=, seg_tensor=, normal_tensor=,
    pc_obj_tensor=, pc_cam_tensor=), filling the caller's [H,W,4] float CUDA tensors from one rast_render_scene call.
    `model_paths` may also be Model3D objects (rendered with whatever shading attributes they were made with).

    Layouts, as the reference leaves its tensors: rows top to bottom (after its torch.flip) for image, seg, pc_obj and
    pc_cam; normal_tensor, which the reference does not flip, bottom to top.  image: BGR with to_bgr, times 255 with
    to_255 (alpha included), alpha 1; pc_obj and normal: alpha 1; everything 0 on background.  pc_cam_tensor[..., 3] is
    the coverage and seg_tensor[..., 0] the instance index + 1, its other channels left as they are.  The light
    position and colour persist across calls, like set_light_pos / set_light_color.

    render(background=): a uint8 [H,W,3] or [H,W] image (NumPy or tensor; 2-D is replicated to three channels, as PIL's
    convert("RGB") does) shown where no instance covers a pixel, as the reference's im2Texture quad: there image_tensor
    holds v / 255 per channel in the given order, then the same to_bgr swap and to_255 scaling as shaded pixels, alpha 1.
    Covered pixels are unchanged.  It fills image_tensor only: depth, seg, pc_obj, pc_cam and normal are those of the
    render without it.  Unlike the reference, which resamples a background of another size through its mip chain, a
    size other than the render's raises ValueError; any dtype but uint8 raises NotImplementedError, as
    PIL.Image.fromarray refuses those."""

    def __init__(self, model_paths, K=None, model_ids=None, texture_paths=None, model_colors=None, width=640, height=480,
                 gpu_id=None, render_marker=False, vertex_scale=1.0, znear=0.25, zfar=6.0, model_loadfn=None,
                 use_cache=False, cad_model_colors=None, device="cuda"):
        """egl_renderer_v3.py:50-67.  model_ids keys the models (default 0..n-1); gpu_id picks cuda:gpu_id; use_cache
        has nothing to cache here.  model_colors (the seg_tensor instance colours), render_marker and
        model_loadfn="pyassimp" raise NotImplementedError."""
        for name, bad in (("model_colors", model_colors is not None), ("render_marker", bool(render_marker)),
                          ("model_loadfn", model_loadfn not in (None, "pysixd"))):
            if bad:
                raise NotImplementedError(f"EGLRenderer: {name} is not supported")
        if gpu_id is not None:
            device = "cuda:%d" % gpu_id
        ms = list(model_paths)
        if ms and isinstance(ms[0], (str, bytes)) or (ms and hasattr(ms[0], "__fspath__")):
            for p in ms:
                if not str(os.fspath(p)).lower().endswith(".ply"):
                    raise NotImplementedError(f"EGLRenderer: {p}: only PLY models; materialed (collada / obj) models "
                                              "are not supported")
            self.models = load_models(ms, scale_to_meter=vertex_scale, device=device, texture_paths=texture_paths,
                                      shading=True, cad_model_colors=cad_model_colors)
        else:
            if (texture_paths is not None and any(texture_paths)) or cad_model_colors is not None:
                raise ValueError("EGLRenderer: texture_paths / cad_model_colors need model paths; give "
                                 "Model3D(..., texture=, colors=) instead")
            self.models = ms
        if model_ids is not None:
            if len(model_ids) != len(self.models):
                raise ValueError(f"EGLRenderer: {len(model_ids)} model_ids for {len(self.models)} models")
            self.models = dict(zip(model_ids, self.models))
        self.K = None if K is None else np.asarray(K, np.float32)
        self.width, self.height, self.znear, self.zfar = width, height, znear, zfar
        self.device = torch.device(device)
        self.lightpos = [0, 0, 0]        # egl_renderer_v3.py:132-133
        self.lightcolor = [1, 1, 1]

    def set_light_pos(self, light):
        self.lightpos = light

    def set_light_color(self, color):
        self.lightcolor = color

    def render(self, obj_ids, poses, K=None, to_bgr=True, to_255=True, rot_type="mat", instance_colors=None,
               light_pos=None, light_color=None, image_tensor=None, seg_tensor=None, normal_tensor=None,
               pc_obj_tensor=None, pc_cam_tensor=None, phong=None, extents=None, gt_extents=None, background=None):
        """Fills the given [H,W,4] tensors (see the class) and returns depth [H,W].  `phong` is accepted and has no
        effect: shader_textureless_texture reads those weights only in its disabled aae_phong branch."""
        if background is not None and background.dtype not in (np.uint8, torch.uint8):
            raise NotImplementedError(f"EGLRenderer.render: background of dtype {background.dtype} is not supported "
                                      "(uint8 only)")
        for name, val in (("instance_colors", instance_colors), ("extents", extents), ("gt_extents", gt_extents)):
            if val is not None:
                raise NotImplementedError(f"EGLRenderer.render: {name} is not supported")
        if rot_type != "mat":
            raise NotImplementedError(f"EGLRenderer.render: rot_type={rot_type!r} is not supported (only 'mat')")
        if isinstance(obj_ids, int):
            obj_ids = [obj_ids]
        if isinstance(poses, np.ndarray) and poses.ndim == 2:
            poses = [poses]
        if K is not None and image_tensor is not None:
            self.height, self.width = int(image_tensor.shape[0]), int(image_tensor.shape[1])
        if light_pos is not None:
            self.set_light_pos(light_pos)
        if light_color is not None:
            self.set_light_color(light_color)
        Kuse = self.K if K is None else np.asarray(K, np.float32)
        H, W = self.height, self.width
        obj_ids, poses = list(obj_ids), list(poses)
        if len(poses) != len(obj_ids):
            raise ValueError(f"EGLRenderer.render: {len(obj_ids)} obj_ids but {len(poses)} poses")
        P = np.zeros((len(obj_ids), 3, 4), np.float32)
        for k, pose in enumerate(poses):
            P[k] = np.asarray(pose, np.float32)[:3, :4]
        ids = torch.tensor([self.models[o].mesh_id for o in obj_ids], dtype=torch.int32).to(self.device)
        outputs = [k for k, t in (("pc_cam", pc_cam_tensor), ("pc_obj", pc_obj_tensor), ("normal", normal_tensor),
                                  ("image", image_tensor), ("seg", seg_tensor)) if t is not None]
        bg = None
        if background is not None:
            bg = torch.as_tensor(background)
            if bg.ndim == 2:
                bg = bg[:, :, None].expand(bg.shape[0], bg.shape[1], 3)
            if tuple(bg.shape) != (H, W, 3):
                raise ValueError(f"EGLRenderer.render: background must be [{H},{W},3] or [{H},{W}] (the render's size), "
                                 f"got {tuple(np.shape(background))}")
            bg = bg.to(self.device).contiguous()
        r = render_scene(ids, torch.from_numpy(P).to(self.device), torch.from_numpy(np.asarray(Kuse, np.float32)), H, W,
                         self.znear, self.zfar, self.lightpos, self.lightcolor, outputs, background=bg)
        depth = r["depth"]
        if pc_cam_tensor is not None:
            pc_cam_tensor[..., :3] = r["pc_cam"]
            if pc_cam_tensor.shape[-1] > 3:
                pc_cam_tensor[..., 3] = (depth > 0).float()
        if seg_tensor is not None:
            seg_tensor[..., 0] = r["seg"]
        if pc_obj_tensor is not None:
            pc_obj_tensor[..., :3] = r["pc_obj"]
            if pc_obj_tensor.shape[-1] > 3:
                pc_obj_tensor[..., 3] = 1.0
        if normal_tensor is not None:
            normal_tensor[..., :3] = torch.flip(r["normal"], (0,))
            if normal_tensor.shape[-1] > 3:
                normal_tensor[..., 3] = 1.0
        if image_tensor is not None:
            image_tensor[..., :3] = r["image"][..., [2, 1, 0]] if to_bgr else r["image"]
            if image_tensor.shape[-1] > 3:
                image_tensor[..., 3] = 1.0
            if to_255:
                image_tensor.mul_(255)
        return depth
