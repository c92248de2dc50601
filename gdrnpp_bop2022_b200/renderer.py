"""CUDA depth rasteriser + fast depth refinement behind the reference's renderer / evaluator surfaces.

Mirrors:
  * lib/render_vispy/renderer.py  Renderer(size, cam).{clear, set_cam, draw_model, finish} -> (rgb, depth)
    (the renderer fast depth refine uses: engine/gdrn_evaluator.py:64-84,520-526; demo/predictor_gdrn.py:100-109)
  * lib/egl_renderer/egl_renderer_v3.py  EGLRenderer.render(obj_ids, poses, K=, pc_cam_tensor=) (depth = pc_cam[...,2])
  * GDRN_Evaluator.process_depth_refine (engine/gdrn_evaluator.py:461-573) == GdrnPredictor.process_depth_refine
    (demo/predictor_gdrn.py:195-286), batched over ROIs on the GPU.
  * get_out_mask / get_out_coor (engine/engine_utils.py:295-333), get_K_crop_resize (core/utils/camera_geometry.py:6-21)
No GL / EGL anywhere; no CPU fallback.
"""
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
    render; without it each mesh's vertex colours, or grey 0.5 for a mesh uploaded without them.  Depth and coverage
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
    colors: optional per-vertex RGB [V,3] in [0,1], which render_meshes_rgb interpolates."""

    def __init__(self, vertices, faces, device="cuda", colors=None):
        v = torch.as_tensor(np.ascontiguousarray(vertices, np.float32))
        f = torch.as_tensor(np.ascontiguousarray(faces, np.int32))
        c = None
        if colors is not None:
            c = torch.as_tensor(np.ascontiguousarray(colors, np.float32))
            if tuple(c.shape) != (v.shape[0], 3):
                raise _lib.GdrnError(f"Model3D: colors must be [V,3] = [{v.shape[0]},3], got {tuple(c.shape)}")
        with torch.cuda.device(device):   # the registry lives on the device current at the upload
            mid = _lib.lib().rast_upload_mesh_ex(_lib.ptr(v), int(v.shape[0]), _lib.ptr(f), int(f.shape[0]), _lib.ptr(c))
        if mid < 0:
            raise _lib.GdrnError(f"rast_upload_mesh failed (code {mid}): {_lib.last_error()}")
        self.mesh_id = mid
        self.vertices = v.to(device)
        self.faces = f.to(device)


def load_models(model_paths, scale_to_meter=1.0, device="cuda", **_):
    """lib/render_vispy/model3d.py:load_models surface: PLY paths -> Model3D list (vertices * scale_to_meter)."""
    from .ply import load_ply

    out = []
    for p in model_paths:
        m = load_ply(p, vertex_scale=scale_to_meter)
        if "faces" not in m:
            raise ValueError(f"{p}: the rasteriser needs a triangle mesh (no face element)")
        out.append(Model3D(m["pts"], m["faces"], device=device))
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


class EGLRenderer:
    """lib/egl_renderer/egl_renderer_v3.py:EGLRenderer surface (:838-857, 1183-1228) for the geometry outputs:
    EGLRenderer(model_paths, K=, width=, height=, vertex_scale=, znear=, zfar=) and
    render(obj_ids, poses, K=, pc_cam_tensor=, seg_tensor=) writing camera-space xyz (float-exact per fragment, like the
    interpolated varying of shader_textureless_texture.vs:36) into the caller's [H,W,4] CUDA tensor.  `model_paths` may
    also be Model3D objects.  Colour / normal / object-space outputs are not rendered."""

    def __init__(self, model_paths, K=None, width=640, height=480, vertex_scale=1.0, znear=0.25, zfar=6.0, device="cuda", **_):
        ms = list(model_paths)
        if ms and isinstance(ms[0], (str, bytes)) or (ms and hasattr(ms[0], "__fspath__")):
            self.models = load_models(ms, scale_to_meter=vertex_scale, device=device)
        else:
            self.models = ms
        self.K = None if K is None else np.asarray(K, np.float32)
        self.width, self.height, self.znear, self.zfar = width, height, znear, zfar
        self.device = torch.device(device)

    def render(self, obj_ids, poses, K=None, pc_cam_tensor=None, seg_tensor=None, **_):
        """Writes camera-space xyz into pc_cam_tensor[..., :3] ([H,W,4] float CUDA, like the reference) and returns depth."""
        Kuse = self.K if K is None else np.asarray(K, np.float32)
        Kt = torch.from_numpy(Kuse)[None].to(self.device)
        depth = torch.zeros((self.height, self.width), device=self.device)
        xyz = torch.zeros((self.height, self.width, 3), device=self.device)
        seg = torch.zeros((self.height, self.width), device=self.device)
        for k, (oid, pose) in enumerate(zip(obj_ids, poses)):
            m = self.models[oid]
            p = torch.as_tensor(np.asarray(pose, np.float32)[:3, :4])[None].to(self.device)
            d, x = render_depth(m, p, Kt, self.height, self.width, self.znear, self.zfar, return_xyz=True)
            upd = (d[0] > 0) & ((depth == 0) | (d[0] < depth))
            depth = torch.where(upd, d[0], depth)
            xyz = torch.where(upd[..., None], x[0], xyz)
            seg = torch.where(upd, torch.full_like(seg, float(k + 1)), seg)
        if pc_cam_tensor is not None:
            pc_cam_tensor[..., :3] = xyz
            if pc_cam_tensor.shape[-1] > 3:
                pc_cam_tensor[..., 3] = (depth > 0).float()
        if seg_tensor is not None:
            seg_tensor[..., 0] = seg
        return depth
