"""f64 NumPy restatement of the scene render's attribute outputs (csrc/raster.cu: rast_render_scene), built on
oracle/raster_oracle.py for visibility.

The n instances are concatenated into one triangle soup in call order (camera-space points, f64), so the rasteriser's
"lower face index wins a depth tie" is "the earlier instance wins".  At each covered pixel the winner's
perspective-correct barycentrics b_k = (w_k / Z_k) / sum(w / Z) (w the screen-space barycentrics at the pixel centre)
interpolate what shader_textureless_texture.vs passes on, with the view matrix at identity:
  pc_obj = sum b_k x_k;  N = sum b_k normalize(R n_k) (not renormalised);  normal = 0.5 N + 0.5;
  FragPos = sum b_k P_k;  diff = max(dot(N, normalize(light - FragPos)), 0);
  image = min(colour (diff + 0.2) light_colour, 1)                            (textureless)
        = min(texture (diff light_colour mat_diffuse + mat_ambient light_colour), 1)   (textured)
Texture: GL_LINEAR_MIPMAP_LINEAR, clamp to edge.  mip_chain halves each dimension (floor, at least 1) with a 2x2 box
filter rounded to nearest, (a + b + c + d + 2) >> 2; lod() is log2 of the larger screen-space derivative length of
(s w0, t h0), the derivatives taken analytically from the triangle's perspective-correct interpolation.
"""
import numpy as np

from oracle import raster_oracle as RO

CAD_COLOR = np.array([223.0, 214.0, 205.0]) / 255.0


def mip_chain(tex):
    """tex [h,w,3] u8 -> list of levels [h_l,w_l,3] u8, down to 1 x 1."""
    levels = [np.asarray(tex, np.uint8)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        s = levels[-1].astype(np.int64)
        h, w = s.shape[:2]
        dh, dw = max(h // 2, 1), max(w // 2, 1)
        y0 = np.minimum(2 * np.arange(dh), h - 1); y1 = np.minimum(2 * np.arange(dh) + 1, h - 1)
        x0 = np.minimum(2 * np.arange(dw), w - 1); x1 = np.minimum(2 * np.arange(dw) + 1, w - 1)
        acc = s[y0][:, x0] + s[y0][:, x1] + s[y1][:, x0] + s[y1][:, x1]
        levels.append(((acc + 2) >> 2).astype(np.uint8))
    return levels


def bilinear(level, s, t):
    """GL_LINEAR with clamp to edge on one level [h,w,3] u8 at (s, t) arrays -> [...,3] in [0,1]; row 0 is t = 0."""
    h, w = level.shape[:2]
    x, y = np.asarray(s, np.float64) * w - 0.5, np.asarray(t, np.float64) * h - 0.5
    fx, fy = np.floor(x), np.floor(y)
    a, b = (x - fx)[..., None], (y - fy)[..., None]
    i0 = np.clip(fx, 0, w - 1).astype(np.int64); i1 = np.clip(fx + 1, 0, w - 1).astype(np.int64)
    j0 = np.clip(fy, 0, h - 1).astype(np.int64); j1 = np.clip(fy + 1, 0, h - 1).astype(np.int64)
    T = level.astype(np.float64) / 255.0
    return (1 - a) * (1 - b) * T[j0, i0] + a * (1 - b) * T[j0, i1] + (1 - a) * b * T[j1, i0] + a * b * T[j1, i1]


def lod(chain, dsdx, dtdx, dsdy, dtdy):
    h0, w0 = chain[0].shape[:2]
    rx = np.hypot(dsdx * w0, dtdx * h0)
    ry = np.hypot(dsdy * w0, dtdy * h0)
    with np.errstate(divide="ignore"):
        return np.log2(np.maximum(rx, ry))


def sample(chain, s, t, lam):
    """GL_LINEAR_MIPMAP_LINEAR (GL_LINEAR magnification) at lod lam: lam <= 0 level 0, lam >= q level q, otherwise
    floor(lam) and floor(lam) + 1 blended by frac(lam)."""
    s, t, lam = (np.asarray(a, np.float64) for a in (s, t, lam))
    q = len(chain) - 1
    out = np.zeros(s.shape + (3,))
    mag = ~(lam > 0)
    out[mag] = bilinear(chain[0], s[mag], t[mag])
    top = (lam >= q) & ~mag
    out[top] = bilinear(chain[q], s[top], t[top])
    mid = ~mag & ~top
    d1 = np.floor(lam[mid]).astype(np.int64)
    fr = (lam[mid] - d1)[:, None]
    sm, tm = s[mid], t[mid]
    res = np.zeros(sm.shape + (3,))
    for d in np.unique(d1):
        k = d1 == d
        res[k] = (1 - fr[k]) * bilinear(chain[d], sm[k], tm[k]) + fr[k] * bilinear(chain[d + 1], sm[k], tm[k])
    out[mid] = res
    return out


def render_scene(meshes, poses, K, H, W, znear, zfar, light_pos=(0, 0, 0), light_color=(1, 1, 1),
                 mat_diffuse=(0.6, 0.6, 0.6), mat_ambient=(0.05, 0.05, 0.05)):
    """meshes: one dict per instance with 'verts' [V,3], 'faces' [F,3] and optional 'normals', 'colors', 'uvs',
    'texture' ([h,w,3] u8, row 0 at t = 0); poses [n,3,4].  -> dict of depth, seg (instance + 1), pc_cam, pc_obj,
    normal, image ([H,W,3] RGB), lod ([H,W], NaN where untextured) and ambiguous [H,W] (raster_oracle's mask)."""
    K = np.asarray(K, np.float64)
    pts, tris, inst, base = [], [], [], 0
    for r, (m, P) in enumerate(zip(meshes, poses)):
        pts.append(RO.camera_points(m["verts"], P))
        tris.append(np.asarray(m["faces"], np.int64) + base)
        inst.append(np.full(len(m["faces"]), r))
        base += len(m["verts"])
    cam = np.concatenate(pts)
    faces = np.concatenate(tris)
    inst = np.concatenate(inst)
    vstart = np.cumsum([0] + [len(m["verts"]) for m in meshes])
    ident = np.hstack([np.eye(3), np.zeros((3, 1))])
    ras = RO.rasterize(cam, faces, ident, K, H, W, znear, zfar)
    face = ras["face"]
    cov = face >= 0
    out = {"depth": ras["depth"], "ambiguous": ras["ambiguous"], "pc_cam": ras["xyz"],
           "seg": np.where(cov, inst[np.maximum(face, 0)] + 1, 0).astype(np.float64)}
    for k in ("pc_obj", "normal", "image"):
        out[k] = np.zeros((H, W, 3))
    out["lod"] = np.full((H, W), np.nan)
    rr, cc = np.nonzero(cov)
    f = face[rr, cc]
    sx, sy = cc + 0.5, rr + 0.5
    Pc = cam[faces[f]]                                   # [m,3,3] camera points
    u = (K[0, 0] * Pc[..., 0] + K[0, 1] * Pc[..., 1]) / Pc[..., 2] + K[0, 2]
    v = K[1, 1] * Pc[..., 1] / Pc[..., 2] + K[1, 2]
    A = (u[:, 1] - u[:, 0]) * (v[:, 2] - v[:, 0]) - (u[:, 2] - u[:, 0]) * (v[:, 1] - v[:, 0])
    w0 = ((u[:, 1] - sx) * (v[:, 2] - sy) - (u[:, 2] - sx) * (v[:, 1] - sy)) / A
    w1 = ((u[:, 2] - sx) * (v[:, 0] - sy) - (u[:, 0] - sx) * (v[:, 2] - sy)) / A
    w = np.stack([w0, w1, 1 - w0 - w1], 1)
    iz = 1.0 / Pc[..., 2]
    izp = (w * iz).sum(1)
    b = w * iz / izp[:, None]
    gx = np.stack([(v[:, 1] - v[:, 2]) / A, (v[:, 2] - v[:, 0]) / A], 1)
    gx = np.concatenate([gx, -gx.sum(1, keepdims=True)], 1)
    gy = np.stack([(u[:, 2] - u[:, 1]) / A, (u[:, 0] - u[:, 2]) / A], 1)
    gy = np.concatenate([gy, -gy.sum(1, keepdims=True)], 1)
    lp, lc = np.asarray(light_pos, np.float64), np.asarray(light_color, np.float64)
    md, ma = np.asarray(mat_diffuse, np.float64), np.asarray(mat_ambient, np.float64)
    for r, m in enumerate(meshes):
        sel = inst[f] == r
        if not sel.any():
            continue
        vi = faces[f[sel]] - vstart[r]                   # [k,3] local vertex indices
        bs = b[sel]
        X = np.asarray(m["verts"], np.float64)
        out["pc_obj"][rr[sel], cc[sel]] = np.einsum("kj,kjc->kc", bs, X[vi])
        R = np.asarray(poses[r], np.float64)[:, :3]
        N = np.zeros((len(vi), 3))
        if m.get("normals") is not None:
            nc = np.asarray(m["normals"], np.float64) @ R.T
            ln = np.linalg.norm(nc, axis=1, keepdims=True)
            nc = np.where(ln > 0, nc / np.where(ln > 0, ln, 1.0), 0.0)
            N = np.einsum("kj,kjc->kc", bs, nc[vi])
        out["normal"][rr[sel], cc[sel]] = 0.5 * N + 0.5
        frag = np.einsum("kj,kjc->kc", bs, Pc[sel])
        L = lp - frag
        L = L / np.linalg.norm(L, axis=1, keepdims=True)
        diff = np.maximum((N * L).sum(1), 0.0)[:, None]
        if m.get("texture") is not None:
            uv = np.asarray(m["uvs"], np.float64)[vi]       # [k,3,2]
            st = np.einsum("kj,kjc->kc", bs, uv)
            izs, izps = iz[sel], izp[sel]
            d = uv - st[:, None, :]
            dx = np.einsum("kj,kjc->kc", gx[sel] * izs, d) / izps[:, None]
            dy = np.einsum("kj,kjc->kc", gy[sel] * izs, d) / izps[:, None]
            chain = m.get("chain") or mip_chain(m["texture"])
            lam = lod(chain, dx[:, 0], dx[:, 1], dy[:, 0], dy[:, 1])
            out["lod"][rr[sel], cc[sel]] = lam
            col = sample(chain, st[:, 0], st[:, 1], lam) * (diff * lc * md + ma * lc)
        else:
            vc = CAD_COLOR[None, None, :] if m.get("colors") is None else np.asarray(m["colors"], np.float64)[vi]
            col = np.einsum("kj,kjc->kc", bs, np.broadcast_to(vc, vi.shape + (3,))) * (diff * lc + 0.2 * lc)
        out["image"][rr[sel], cc[sel]] = np.minimum(col, 1.0)
    return out
