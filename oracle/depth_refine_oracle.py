"""f64 restatement of the fast depth refine (engine/gdrn_evaluator.py:515-561, engine_utils.get_out_mask), one
function per stage, on the f32 inputs the kernel receives.

One step: mask normalisation -> weights w (||xyz|| or the coor-z (R xyz)_z, times the mask, zero where the render or
the sensor has no depth) -> w / sum(w) -> selection w / sum > thresh * max(w / sum) -> median of sensor - render over
the selection -> weighted centroid (y, x) -> ray K^-1 (x, y, 1) / z -> t += ray * median.

Where the kernel departs from the reference it is followed here, and the departure is named: an empty selection (a
constant L1 mask makes the cut NaN; thresh >= 1 selects nothing) leaves t unchanged where the reference's
np.median([]) would give NaN.
"""
import numpy as np

SEL_BAND = 2.0 ** -21   # relative band around the cut inside which f32 rounding decides the selection (8 f32 ulps)


def out_mask(raw, mode):
    """get_out_mask in f64: 0 = already normalised (identity), 1 = per-ROI min-max (the L1 head; a constant mask gives
    0 / 0 = NaN), 2 = sigmoid (BCE / RW_BCE / dice heads)."""
    m = np.asarray(raw, np.float64)
    if mode == 0:
        return m.copy()
    if mode == 1:
        with np.errstate(invalid="ignore", divide="ignore"):
            return (m - m.min()) / (m.max() - m.min())
    if mode == 2:
        return 1.0 / (1.0 + np.exp(-m))
    raise ValueError(mode)


def weights(xyz, mask, ren, sensor, R=None, weight_mode=0):
    """xyz [3,hw,hw], mask [hw,hw] normalised, ren / sensor [hw,hw] -> w [hw,hw] f64: ||xyz|| * mask (weight_mode 0)
    or (R xyz)_z * mask (1, TEST.USE_COOR_Z_REFINE), 0 wherever the render or the sensor has no depth."""
    x = np.asarray(xyz, np.float64)
    if weight_mode == 0:
        q = np.sqrt((x * x).sum(0))
    else:
        r = np.asarray(R, np.float64)[2]
        q = r[0] * x[0] + r[1] * x[1] + r[2] * x[2]
    valid = (np.asarray(ren) > 0) & (np.asarray(sensor) > 0)
    with np.errstate(invalid="ignore"):
        return np.where(valid, q * np.asarray(mask, np.float64), 0.0)


def normalise_and_select(w, thresh, band=SEL_BAND):
    """w [hw,hw] -> dict: sum, max and min (over all pixels, zero included), wn = w / sum, cut = max(wn) * thresh,
    sel = wn > cut, and amb, the pixels whose wn lies within `band` (relative) of the cut, where rounding decides.
    A zero sum returns sum 0 and nothing else (the pose is unchanged)."""
    w = np.asarray(w, np.float64)
    s = float(np.sum(w, dtype=np.float64))
    out = {"sum": s, "max": max(0.0, float(np.nanmax(w, initial=0.0))), "min": min(0.0, float(np.nanmin(w, initial=0.0)))}
    if s == 0.0:
        return out
    with np.errstate(invalid="ignore"):
        wn = w / s
        cut = float(np.max(wn)) * thresh
        out.update(wn=wn, cut=cut, sel=wn > cut, amb=np.abs(wn - cut) <= band * abs(cut))
    return out


def median(diffs):
    """np.median semantics: the middle element, or for an even count the mean of the two middle elements, formed in
    the dtype of `diffs` (f32 for the sensor - render diffs, as the reference); an empty selection gives NaN."""
    d = np.sort(np.asarray(diffs).ravel())
    n = len(d)
    if n == 0:
        return float("nan")
    return d[n // 2] if n % 2 else (d[n // 2 - 1] + d[n // 2]) / d.dtype.type(2)


def centroid(wn):
    """Weighted pixel centroid (y, x) = sum(wn * (row, col))."""
    wn = np.asarray(wn, np.float64)
    rows, cols = np.indices(wn.shape, dtype=np.float64)
    return float(np.sum(wn * rows)), float(np.sum(wn * cols))


def ray(K, c):
    """K^-1 (x, y, 1) normalised by its z, from the centroid c = (y, x)."""
    r = np.linalg.inv(np.asarray(K, np.float64)) @ np.array([c[1], c[0], 1.0])
    return r / r[2]


def step(xyz, raw_mask, ren, sensor, K, t, R=None, mask_mode=1, weight_mode=0, thresh=0.8, band=SEL_BAND):
    """One refine step -> (t_new f64 [3], stages dict).  stages holds every intermediate (mask, w, the
    normalise_and_select dict, diffs, med, centroid, ray); 'changed' says whether t moved (False for a zero sum or an
    empty selection, the kernel's behaviour for the latter)."""
    t = np.asarray(t, np.float64)
    m = out_mask(raw_mask, mask_mode)
    w = weights(xyz, m, ren, sensor, R, weight_mode)
    st = {"mask": m, "w": w, "ns": normalise_and_select(w, thresh, band), "changed": False}
    ns = st["ns"]
    if ns["sum"] == 0.0 or not ns["sel"].any():
        return t.copy(), st
    diffs = np.asarray(sensor, np.float32)[ns["sel"]] - np.asarray(ren, np.float32)[ns["sel"]]   # f32, as the reference
    st.update(diffs=diffs, med=median(diffs), centroid=centroid(ns["wn"]))
    st["ray"] = ray(K, st["centroid"])
    st["changed"] = True
    return t + st["ray"] * st["med"], st


def replay(render_fn, xyz, raw_mask, sensor, K, R, t, iters=2, **kw):
    """`iters` x (ren = render_fn(R, t) -> step): the refine loop of gdrn_evaluator.py:515-561 for one ROI.  Returns
    the final t and the stages of every step."""
    t = np.asarray(t, np.float64)
    stages = []
    for _ in range(iters):
        ren = render_fn(R, t)
        t, st = step(xyz, raw_mask, ren, sensor, K, t, R=R, **kw)
        stages.append(st)
    return t, stages
