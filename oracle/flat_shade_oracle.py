"""f64 NumPy restatement of renderer_py's flat shading (lib/pysixd/renderer_py.py:52-75, light at the eye origin,
ambient 0.5), given the triangle seen at each pixel.

Per pixel with triangle f: the screen barycentrics of the pixel centre (c + 0.5, r + 0.5) in f64, made
perspective-correct; L = normalize(sum(b_k * normalize(-P_k))); n = the camera-frame face normal turned toward the
viewer (dot(n, P_0) <= 0); light_w = min(0.5 + max(dot(L, n), 0), 1); value = light_w * colour * 255 (unrounded).
Colour: the uniform colour, else the interpolated vertex colours, else 0.5.
"""
import numpy as np


def flat_shade(verts, faces, pose, K, tri_ids, color=None, vert_colors=None):
    """verts [V,3], faces [F,3], pose [3,4], K [3,3], tri_ids [H,W] (-1 = background) -> [H,W,3] f64 in [0, 255]."""
    V = np.asarray(verts, np.float64)
    P = V @ np.asarray(pose, np.float64)[:, :3].T + np.asarray(pose, np.float64)[:, 3]
    K = np.asarray(K, np.float64)
    H, W = tri_ids.shape
    out = np.zeros((H, W, 3))
    rows, cols = np.nonzero(tri_ids >= 0)
    f = np.asarray(faces)[tri_ids[rows, cols]]                      # [m,3] vertex indices
    Pk = P[f]                                                        # [m,3,3]
    u = (K[0, 0] * Pk[..., 0] + K[0, 1] * Pk[..., 1]) / Pk[..., 2] + K[0, 2]
    v = K[1, 1] * Pk[..., 1] / Pk[..., 2] + K[1, 2]
    sx, sy = cols + 0.5, rows + 0.5
    area = (u[:, 1] - u[:, 0]) * (v[:, 2] - v[:, 0]) - (u[:, 2] - u[:, 0]) * (v[:, 1] - v[:, 0])
    w0 = ((u[:, 1] - sx) * (v[:, 2] - sy) - (u[:, 2] - sx) * (v[:, 1] - sy)) / area
    w1 = ((u[:, 2] - sx) * (v[:, 0] - sy) - (u[:, 0] - sx) * (v[:, 2] - sy)) / area
    w = np.stack([w0, w1, 1.0 - w0 - w1], axis=1) / Pk[..., 2]
    b = w / w.sum(axis=1, keepdims=True)                              # perspective-correct weights
    Lv = -Pk / np.linalg.norm(Pk, axis=2, keepdims=True)
    L = np.einsum("mk,mkc->mc", b, Lv)
    L /= np.linalg.norm(L, axis=1, keepdims=True)
    n = np.cross(Pk[:, 1] - Pk[:, 0], Pk[:, 2] - Pk[:, 0])
    n *= np.where(np.einsum("mc,mc->m", n, Pk[:, 0]) > 0, -1.0, 1.0)[:, None]
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    lw = np.minimum(0.5 + np.maximum(np.einsum("mc,mc->m", L, n), 0.0), 1.0)
    if color is not None:
        col = np.broadcast_to(np.asarray(color, np.float64), (len(rows), 3))
    elif vert_colors is not None:
        col = np.einsum("mk,mkc->mc", b, np.asarray(vert_colors, np.float64)[f])
    else:
        col = np.full((len(rows), 3), 0.5)
    out[rows, cols] = lw[:, None] * col * 255.0
    return out
