"""Host restatements of the vis_poses_full scripts' pixel work (core/gdrn_modeling/tools/*/..._vis_poses_full.py),
the references gdrn_vis_gray3 and gdrn_vis_outlines are tested against and the host arm of bench_vis_poses_full.py."""
import numpy as np


def get_edge(mask, bw=3):
    """lib/utils/mask_utils.py:get_edge(mask, bw, out_channel=1) != 0 for a 2-D 0/1 mask."""
    m = np.asarray(mask)
    e = np.zeros(m.shape, bool)
    e[:-bw, :] |= (m[:-bw, :] == 1) & (m[bw:, :] == 0)
    e[bw:, :] |= (m[bw:, :] == 1) & (m[:-bw, :] == 0)
    e[:, :-bw] |= (m[:, :-bw] == 1) & (m[:, bw:] == 0)
    e[:, bw:] |= (m[:, bw:] == 1) & (m[:, :-bw] == 0)
    return e


def mask2bbox_xyxy(mask):
    """lib/utils/mask_utils.py:mask2bbox_xyxy: bottom-right pixel included."""
    ys, xs = np.nonzero(mask)[:2]
    return [int(xs.min()), int(ys.min()), int(xs.max()), int(ys.max())]


def bgr2gray3(bgr):
    """cv2.cvtColor(BGR2GRAY) on u8 stacked three times: (3735 b + 19235 g + 9798 r + 16384) >> 15."""
    b, g, r = (bgr[..., c].astype(np.int64) for c in range(3))
    y = ((3735 * b + 19235 * g + 9798 * r + 16384) >> 15).astype(np.uint8)
    return np.stack([y, y, y], axis=-1)


def ren_bgr(image_rgb):
    """Step 2 of the scripts after the render: image_tensor = bgr(image) * 255 in f32 (EGLRenderer's to_bgr, to_255),
    then (image_tensor[..., :3] + 0.5).astype(uint8), for render_scene's RGB "image" [H,W,3] f32."""
    t = np.ascontiguousarray(np.asarray(image_rgb, np.float32)[..., ::-1]) * np.float32(255)
    return (t + np.float32(0.5)).astype(np.uint8)


def composite(image_rgb, gt_masks, est_masks, bw=3):
    """Step 3, the scripts' loop literally: ren_bgr, then each GT mask's edges painted blue, then each estimate's green."""
    out = ren_bgr(image_rgb)
    for m in gt_masks:
        out[get_edge(m, bw)] = (255, 0, 0)
    for m in est_masks:
        out[get_edge(m, bw)] = (0, 255, 0)
    return out
