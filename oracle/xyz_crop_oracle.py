"""fp64 NumPy restatement of one xyz_crop training target (the *_1_gen_xyz.py scripts' per-instance math).

From a render's depth image and the f32 inputs the scripts use: the inclusive box of depth != 0, the back-projection of
misc.calc_xyz_bp_torch, xyz = R^T (((u - cx) z / fx, (v - cy) z / fy, z) - t) with 0 where z == 0, evaluated in f64,
the crop rounded once to fp16 (round to nearest even, as numpy's astype does it) and the dict mmcv.dump writes.  An
empty render gives full-frame zeros and the box [0, 0, W - 1, H - 1]."""
import numpy as np


def xyz_crop(depth, R, t, K):
    """depth [H,W] (the render, f32), R [3,3], t [3] (metres), K [3,3], each taken as f32 and then widened to f64.
    -> (xyxy [x1, y1, x2, y2] ints, xyz [h,w,3] f64 before rounding, xyz_crop [h,w,3] f16)."""
    depth = np.asarray(depth, np.float32)
    R = np.asarray(R, np.float32).reshape(3, 3).astype(np.float64)
    t = np.asarray(t, np.float32).reshape(3).astype(np.float64)
    K = np.asarray(K, np.float32).reshape(3, 3).astype(np.float64)
    H, W = depth.shape
    ys, xs = np.nonzero(depth != 0)
    if xs.size == 0:
        z = np.zeros((H, W, 3))
        return [0, 0, W - 1, H - 1], z, z.astype(np.float16)
    x1, y1, x2, y2 = int(xs.min()), int(ys.min()), int(xs.max()), int(ys.max())
    z = depth[y1:y2 + 1, x1:x2 + 1].astype(np.float64)
    u = np.arange(x1, x2 + 1, dtype=np.float64)[None, :]
    v = np.arange(y1, y2 + 1, dtype=np.float64)[:, None]
    cam = np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z], axis=-1)
    xyz = (cam - t) @ R            # R^T p for each pixel p
    xyz[z == 0] = 0.0
    return [x1, y1, x2, y2], xyz, xyz.astype(np.float16)


def file_dict(depth, R, t, K):
    """The dict the scripts dump: {"xyz_crop": f16 [h,w,3], "xyxy": [x1, y1, x2, y2]}."""
    xyxy, _, crop = xyz_crop(depth, R, t, K)
    return {"xyz_crop": crop, "xyxy": xyxy}


def fp16_ulp_distance(a, b):
    """Elementwise distance in fp16 units in the last place between two f16 arrays (+0 and -0 are 0 apart)."""
    def ordered(x):
        i = np.asarray(x, np.float16).view(np.int16).astype(np.int32)
        return np.where(i < 0, -(i & 0x7FFF), i)

    return np.abs(ordered(a) - ordered(b))
