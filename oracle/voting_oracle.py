"""ORACLE (test infrastructure, NOT product code): the RANSAC voting driver (core/csrc/ransac_voting/ransac_voting_gpu.py)
restated in NumPy one stage at a time, for tests/test_voting_stages.py.

Hypotheses and votes go through ops_oracle.generate_hypothesis / ops_oracle.voting, which are bit-exact against the
reference's CUDA kernels.  The refit and the covariance are float64.  The voting-distribution ratios and their drop
threshold stay in float32, the dtype the reference computes them in, so that a ratio at the `max - 0.1` boundary is
kept or dropped as the reference decides.

Stages of one image (the reference loops over the batch):
  foreground_weights -> compact -> hypotheses -> counts -> winner -> inliers -> refit
and voting_distribution for estimate_voting_distribution_with_mean.
"""
import numpy as np

from . import ops_oracle as OO

# The refit's singularity rule, the one rv_refit_kernel applies: |det| <= REFIT_SINGULAR_RTOL * max(1, |a00 * a11|)
REFIT_SINGULAR_RTOL = 1e-12


def foreground_weights(mask, semantics):
    """Per-pixel foreground weight of a non-negative mask (values below 256) under each reference driver's reading:
      "byte" -- ransac_voting_layer, `mask[bi].byte()` (:28): the value truncated to an integer, so (0, 1) is
                background and a pixel of value k counts k times in `foreground_num = torch.sum(cur_mask)`;
      "bool" -- ransac_voting_layer_v3, `.to(torch.bool)` (:144): every non-zero value is one pixel;
      "eq1"  -- estimate_voting_distribution_with_mean, `mask[bi] == 1` (:237)."""
    mask = np.asarray(mask)
    if semantics == "byte":
        return np.trunc(mask.astype(np.float64)).astype(np.int64)
    if semantics == "bool":
        return (mask != 0).astype(np.int64)
    if semantics == "eq1":
        return (mask == 1).astype(np.int64)
    raise ValueError(semantics)


def keep_probability(fg, max_num):
    """(subsampled, keep probability): an image whose foreground count exceeds max_num keeps each pixel with probability
    max_num / fg, in float32 as `max_num / foreground_num.float()` (:38-40)."""
    if fg > max_num:
        return True, float(np.float32(max_num) / np.float32(fg))
    return False, 1.0


def compact(keep, vertex):
    """torch.nonzero row-major order, coords[:, [1, 0]] = (x, y), and masked_select of the directions (:43-46).
    keep [h,w] bool (the foreground, or what subsampling left of it), vertex [h,w,vn,2] -> coords [tn,2], direct
    [tn,vn,2] float32."""
    ys, xs = np.nonzero(keep)
    coords = np.stack([xs, ys], 1).astype(np.float32).reshape(-1, 2)
    direct = np.ascontiguousarray(np.asarray(vertex, np.float32)[ys, xs])
    return coords, direct


def compact_image(weights, vertex, min_num, max_num):
    """The compaction stage of an image that is not subsampled: -> (fg, coords, direct), with tn = 0 when fg < min_num.
    Raises for a subsampled image, whose kept set is a random draw."""
    fg = int(np.asarray(weights).sum())
    vn = np.asarray(vertex).shape[2]
    if fg < min_num:
        return fg, np.zeros((0, 2), np.float32), np.zeros((0, vn, 2), np.float32)
    if keep_probability(fg, max_num)[0]:
        raise ValueError("a subsampled image has no deterministic compaction")
    return (fg,) + compact(np.asarray(weights) != 0, vertex)


def pair_indices(idxs, tn):
    """Caller-supplied pixel pairs [hn,vn,2] (non-negative) taken modulo tn, as the layer takes them."""
    return (np.asarray(idxs, np.int64) % max(tn, 1)).astype(np.int32)


def hypotheses(direct, coords, idxs):
    """[hn,vn,2] line intersections of the pairs (zeros for a degenerate pair, and everywhere when tn = 0)."""
    idxs = np.asarray(idxs)
    tn, vn = direct.shape[0], idxs.shape[1]
    if tn == 0:
        return np.zeros((idxs.shape[0], vn, 2), np.float32)
    return OO.generate_hypothesis(direct, coords, pair_indices(idxs, tn))


def counts(direct, coords, hyp, thresh):
    """[hn,vn] int: votes of the tn pixels for every hypothesis (torch.sum(cur_inlier, 2), :62)."""
    if direct.shape[0] == 0:
        return np.zeros(hyp.shape[:2], np.int64)
    return OO.voting(direct, coords, hyp, thresh)[1].astype(np.int64)


def winner(cnt, hyp):
    """Per keypoint: torch.max over the hypotheses (the highest count, the lowest index on ties) and the strict
    `all_win_ratio < cur_win_ratio` update from zero (:63-70): a best count of 0 leaves the winner at (0, 0).
    -> (win_pts [vn,2] float32, index [vn], best count [vn])."""
    vn = cnt.shape[1]
    idx = np.argmax(cnt, axis=0)
    best = cnt[idx, np.arange(vn)]
    win = hyp[idx, np.arange(vn)].astype(np.float32)
    win[best <= 0] = 0.0
    return win, idx, best


def inliers(direct, coords, win, thresh):
    """[vn,tn] uint8: the inlier set of the winners (voting_for_hypothesis(all_win_pts), :85)."""
    if direct.shape[0] == 0:
        return np.zeros((win.shape[0], 0), np.uint8)
    return OO.voting(direct, coords, win[None], thresh)[0][0]


def normal_equations(direct, coords, inl):
    """The 2x2 system of the refit (:80-94) in float64: normal (d.y, -d.x) of every inlier line, ATA [vn,2,2] and ATb
    [vn,2]."""
    d = direct.astype(np.float64)
    n = np.stack([d[:, :, 1], -d[:, :, 0]], -1).transpose(1, 0, 2) * inl[:, :, None]       # [vn,tn,2]
    b = (n * coords.astype(np.float64)[None]).sum(-1)                                      # [vn,tn]
    ata = np.einsum("vti,vtj->vij", n, n)
    atb = (n * b[:, :, None]).sum(1)
    return ata, atb


def refit(direct, coords, inl):
    """Least-squares intersection of each keypoint's inlier lines in float64 -> (pts [vn,2] float64, singular [vn]).
    A singular system takes b_inv's identity fallback (:107-120), pts = ATb.  The reference applies its fallback to
    the whole [vn,2,2] batch of an image when any of its systems is singular (and v1 emits zeros instead); the layer,
    and this restatement, decide per keypoint."""
    ata, atb = normal_equations(direct, coords, inl)
    det = ata[:, 0, 0] * ata[:, 1, 1] - ata[:, 0, 1] * ata[:, 1, 0]
    singular = ~(np.abs(det) > REFIT_SINGULAR_RTOL * np.maximum(1.0, np.abs(ata[:, 0, 0] * ata[:, 1, 1])))
    pts = atb.copy()
    ok = ~singular
    if ok.any():
        pts[ok] = np.linalg.solve(ata[ok], atb[ok][:, :, None])[:, :, 0]
    return pts, singular


def voting_layer(weights, vertex, idxs, thresh, min_num=5, max_num=30000):
    """The whole driver on one image that is not subsampled, with the pixel pairs idxs [hn,vn,2] in place of its
    random_ draw -> dict of every stage."""
    fg, coords, direct = compact_image(weights, vertex, min_num, max_num)
    hyp = hypotheses(direct, coords, idxs)
    cnt = counts(direct, coords, hyp, thresh)
    win, idx, best = winner(cnt, hyp)
    inl = inliers(direct, coords, win, thresh)
    vn = hyp.shape[1]
    pts, singular = refit(direct, coords, inl) if direct.shape[0] else (np.zeros((vn, 2)), np.zeros(vn, bool))
    return dict(fg=fg, tn=direct.shape[0], coords=coords, direct=direct, hyp=hyp, cnt=cnt, win=win, win_idx=idx,
                best=best, inliers=inl, pts=pts, singular=singular)


def voting_distribution(hyp, cnt, tn, mean):
    """estimate_voting_distribution_with_mean (:290-304) from given hypotheses hyp [b,hn,vn,2], counts [b,hn,vn] and
    foreground counts tn [b] around mean [b,vn,2] -> cov [b,vn,2,2] float64.

    ratio = count / tn and the drop threshold max - 0.1 are float32, as in the reference; an image with tn = 0 weighs
    its (zero) hypotheses by 1 (:241-249).  The weighted second moment and its normaliser sum(ratio) + 1e-3 are
    float64."""
    hyp, cnt, tn = np.asarray(hyp), np.asarray(cnt), np.asarray(tn)
    ratio = cnt.astype(np.float32) / np.maximum(tn, 1).astype(np.float32)[:, None, None]
    ratio[tn <= 0] = np.float32(1.0)
    ratio = ratio.transpose(0, 2, 1)                                                      # b,vn,hn
    thresh = ratio.max(2) - np.float32(0.1)
    ratio = np.where(ratio < thresh[:, :, None], np.float32(0.0), ratio).astype(np.float64)
    diff = hyp.transpose(0, 2, 1, 3).astype(np.float64) - np.asarray(mean, np.float64)[:, :, None]   # b,vn,hn,2
    cov = np.einsum("bvhi,bvhj->bvij", diff, diff * ratio[..., None])
    return cov / (ratio.sum(2)[:, :, None, None] + 1e-3)
