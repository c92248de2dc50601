"""Every error type of lib/pysixd/scripts/eval_pose_results_more.py, with the errors as batched GPU calls.

bop_eval.py evaluates the six BOP19 types (vsd, mssd, mspd, ad, add, adi), as the reference's eval_bop19.py does.  This
script is the counterpart of eval_pose_results_more.py: it adds the fourteen other types of that script's table
(eval_calc_errors.py:478-597), one GPU call per error type for all pairs, and reuses bop_eval's loaders, pair
selection, matching, scoring and output files:
  * re / te / rete            pose_error.re, te (against the GT pose itself), deg and cm
  * reS / teS / reteS         re_sym, te_sym: each minimised over the object's symmetry set on its own
  * proj / projS              arp_2d, arp_2d_sym: mean 2D distance of the model points' projections, px
  * ABSadd / ABSadi / ABSad,  add, adi, or ADI for the dataset's symmetric objects and ADD otherwise, in cm and with no
    AUCadd / AUCadi / AUCad   sphere gate (a far-off estimate gets a finite error, not inf)
None of these errors is normalised before thresholding.  VAL.SCRIPT_PATH can point at this file; run by path it takes
bop_eval.py's arguments, and its default --error_types is the reference script's.
"""
import os
import sys

if __package__ in (None, ""):   # run by path, as VAL.SCRIPT_PATH is invoked
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    __package__ = "gdrnpp_bop2022_b200"

import numpy as np

from . import bop_eval

# eval_pose_results_more.py:39-178, in the reference's order
KNOWN_ERROR_TYPES = ("vsd", "mssd", "mspd", "add", "adi", "ad", "ABSadd", "ABSadi", "ABSad", "AUCadd", "AUCadi", "AUCad",
                     "re", "te", "rete", "proj", "reS", "teS", "reteS", "projS")
CORRECT_TH = {
    **bop_eval.CORRECT_TH,
    **{t: [[th] for th in [2]] for t in ("ABSadd", "ABSadi", "ABSad")},                          # cm
    **{t: [[th] for th in np.linspace(10 / 10, 10, num=10)] for t in ("AUCadd", "AUCadi", "AUCad")},   # cm
    **{t: [[th] for th in [2, 5, 10]] for t in ("re", "te", "proj", "reS", "teS", "projS")},   # deg, cm, px
    **{t: [[2, 2], [5, 5], [10, 10]] for t in ("rete", "reteS")},                              # deg and cm
}
DEFAULT_ERROR_TYPES = "mspd,mssd,vsd,reteS,add,adi,teS,reS,projS"


def calc_errors(error_type, dataset, ests, targets, scene_gts, scene_cameras, models_info, models=None, meshes=None,
                load_depth=None, n_top=-1, skip_missing=True, vsd_delta=None, vsd_taus=None, vsd_normalized_by_diameter=True,
                max_bytes=2 << 30):
    """bop_eval.calc_errors for every type of KNOWN_ERROR_TYPES: the BOP19 types go to bop_eval.calc_errors, the others
    are one GPU call for all pairs.  Same arguments and record layout; models (PoseErrorModels) serves every new type."""
    if error_type in bop_eval.ERROR_TYPES:
        return bop_eval.calc_errors(error_type, dataset, ests, targets, scene_gts, scene_cameras, models_info, models,
                                    meshes, load_depth, n_top, skip_missing, vsd_delta, vsd_taus,
                                    vsd_normalized_by_diameter, max_bytes)
    if error_type not in KNOWN_ERROR_TYPES:
        raise ValueError(f"error type {error_type!r} is not supported (supported: {', '.join(KNOWN_ERROR_TYPES)})")
    records, pairs, arrays = bop_eval.error_pairs(ests, targets, scene_gts, scene_cameras, models_info, n_top,
                                                  skip_missing)
    if not pairs:
        return records
    _, R_e, t_e, R_g, t_g, K, obj = arrays
    use_syms = error_type.endswith("S")
    if error_type in ("re", "te", "rete", "reS", "teS", "reteS"):
        re_deg, te_mm = (x.cpu().numpy() for x in bop_eval.rt_errors(models, obj, R_e, t_e, R_g, t_g, use_syms))
        te_cm = te_mm / 10
        errs = {"re": [re_deg], "te": [te_cm], "rete": [re_deg, te_cm]}[error_type.rstrip("S")]
        errs = np.stack(errs, axis=1)
    elif error_type in ("proj", "projS"):
        errs = bop_eval.proj_errors(models, obj, R_e, t_e, R_g, t_g, K, use_syms).cpu().numpy()[:, None]
    else:   # ABS* / AUC*: ADD / ADI in cm, never gated
        kind = error_type[3:]
        use_adi = [kind == "adi" or (kind == "ad" and bop_eval.is_symmetric(dataset, o, models_info[o])) for o in obj]
        errs = (bop_eval.ad(models, obj, R_e, t_e, R_g, t_g, use_adi).cpu().numpy() / 10)[:, None]
    return bop_eval.fill_errors(records, pairs, errs)


def evaluate(error_types, dataset, ests, targets, scene_gts, scene_cameras, scene_gt_infos, models_info, im_width,
             models=None, meshes=None, load_depth=None, n_top=-1, max_bytes=2 << 30, scene_ids=None, obj_ids=None):
    """bop_eval.evaluate over every type of KNOWN_ERROR_TYPES.  -> ({'bop19_average_recall_<type>': AR, ...,
    'bop19_average_recall' when vsd, mssd and mspd are all present}, {type: errors})."""
    return bop_eval.evaluate(error_types, dataset, ests, targets, scene_gts, scene_cameras, scene_gt_infos, models_info,
                             im_width, models, meshes, load_depth, n_top, max_bytes, scene_ids, obj_ids,
                             calc=calc_errors, correct_th=CORRECT_TH)


def parse_args(argv=None):
    return bop_eval.parse_eval_args(argv, "Pose-error evaluation on the GPU, every error type of "
                                    "eval_pose_results_more.py", DEFAULT_ERROR_TYPES, KNOWN_ERROR_TYPES)


def run(args):
    """bop_eval.run over every type of KNOWN_ERROR_TYPES: the same files under the same signatures."""
    return bop_eval.run(args, calc=calc_errors, correct_th=CORRECT_TH)


if __name__ == "__main__":
    run(parse_args())
