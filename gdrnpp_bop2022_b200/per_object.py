"""Per-object deployment: one class-agnostic GDRN_DoubleMask per object, one call for a mixed batch of ROIs.

The reference trains most of its networks per object (configs/gdrn/*SO/**: one ConvNeXt-base with a class-agnostic
head per object) and evaluates one model at a time.  ``PerObjectGDRN`` takes a batch whose ROIs belong to different
objects, sends every ROI to its object's network and returns poses (and maps) in input order:

  * ROIs are grouped by label on the host (``group_rois``); every member runs its sub-batch on its own CUDA stream,
    forked from and joined back into the caller's stream with events, so the small per-member forwards overlap;
  * gathering and scattering are torch indexing on those streams (the 256x256 crop is ~0.8 MB per ROI, small next to
    the forward itself);
  * every forward gets a workspace of its own sub-batch size, so device memory follows the number of ROIs in the
    call, not members x max_batch;
  * with ``use_cuda_graph=True`` every (member, sub-batch size) pair is captured once into a CUDA graph over static
    buffers and replayed on the member's stream: a frame of 5 ROIs of 5 different objects costs 5 graph launches
    instead of ~5 x 150 kernel launches.
"""
import torch

from . import _lib
from .gdrn_model import GDRN_DoubleMask

_INPUTS = ("roi_img", "roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "roi_extents", "resize_ratios")


def group_rois(labels, known):
    """Group ROI indices by label.  ``labels``: 1-D integer sequence or tensor (a device tensor is copied to the host,
    which waits for the work that produces it); ``known``: the labels that have a model.

    Returns ``[(label, idx)]`` in ascending label order, ``idx`` an int64 CPU tensor of the ROIs with that label in
    input order, so that writing every group's results to ``out[idx]`` restores the input order.  Raises ValueError
    naming every label that has no model."""
    lab = torch.as_tensor(labels).detach().to("cpu", torch.int64).reshape(-1)
    present = torch.unique(lab).tolist()
    missing = [u for u in present if u not in known]
    if missing:
        raise ValueError(f"no per-object model for label(s) {missing}; models exist for {sorted(known)}")
    return [(u, torch.nonzero(lab == u).flatten()) for u in present]


class PerObjectGDRN:
    """``{label: GDRN_DoubleMask}`` of class-agnostic members (same precision, one device) behind the forward of one
    model.  ``forward`` takes the arguments of ``GDRN_DoubleMask.forward`` and returns the same dict; ``roi_classes``
    picks each ROI's member."""

    def __init__(self, members, use_cuda_graph=False):
        if not members:
            raise ValueError("PerObjectGDRN needs at least one member model")
        self.members = {}
        for label, m in members.items():
            if not isinstance(m, GDRN_DoubleMask):
                raise TypeError(f"member {label!r} is a {type(m).__name__}, not a GDRN_DoubleMask")
            if m.class_aware:
                raise ValueError(f"member {label!r} has a class-aware head; per-object members are class-agnostic "
                                 "(XYZ/MASK/REGION_CLASS_AWARE false)")
            self.members[int(label)] = m
        ms = list(self.members.values())
        if len({m.precision for m in ms}) != 1:
            raise ValueError("all members must use the same precision, got "
                             f"{sorted({m.precision for m in ms})}")
        if len({m.wants_maps for m in ms}) != 1:
            raise ValueError("all members must agree on returning the geometry maps (TEST.USE_PNP / "
                             "SAVE_RESULTS_ONLY / USE_DEPTH_REFINE)")
        devs = {p.device for m in ms for p in m.parameters()} | {m._engine_device for m in ms if m._engine_device}
        if len(devs) != 1:
            raise ValueError(f"all members must live on one device, got {sorted(map(str, devs))}")
        self.precision = ms[0].precision
        self.wants_maps = ms[0].wants_maps
        self.use_cuda_graph = bool(use_cuda_graph)
        self._streams = {}   # label -> the member's CUDA stream
        self._graphs = {}    # (label, n) -> (static inputs, replay, static outputs)

    def __call__(self, *a, **k):
        return self.forward(*a, **k)

    def _stream(self, label, dev):
        s = self._streams.get(label)
        if s is None:
            s = self._streams[label] = torch.cuda.Stream(device=dev)
        return s

    def release_graphs(self):
        """Drop the captured graphs and their static buffers (the members may then reload weights)."""
        self._graphs.clear()
        for m in self.members.values():
            m.release_graphs()

    def forward(self, x, gt_xyz=None, gt_xyz_bin=None, gt_mask_trunc=None, gt_mask_visib=None, gt_mask_obj=None,
                gt_mask_full=None, gt_region=None, gt_ego_rot=None, gt_points=None, sym_infos=None, gt_trans=None,
                gt_trans_ratio=None, roi_classes=None, roi_coord_2d=None, roi_cams=None, roi_centers=None,
                roi_whs=None, roi_extents=None, resize_ratios=None, do_loss=False, return_raw=False):
        if do_loss:
            raise NotImplementedError("training (do_loss=True) is out of scope of the inference hot path")
        if not x.is_cuda:
            raise _lib.GdrnError("PerObjectGDRN.forward needs CUDA tensors (no CPU fallback)")
        if return_raw and self.use_cuda_graph:
            raise ValueError("return_raw is not part of the captured graphs: use use_cuda_graph=False")
        for name, t in (("roi_classes", roi_classes), ("roi_coord_2d", roi_coord_2d), ("roi_cams", roi_cams),
                        ("roi_centers", roi_centers), ("roi_whs", roi_whs), ("roi_extents", roi_extents),
                        ("resize_ratios", resize_ratios)):
            if t is None:
                raise ValueError(f"{name} is required" + (" (it selects each ROI's model)" if name == "roi_classes" else ""))
        dev = x.device
        B = x.shape[0]
        if tuple(x.shape[1:]) != (3, 256, 256):
            raise ValueError(f"roi_img must be [B,3,256,256], got {tuple(x.shape)}")
        if int(torch.as_tensor(roi_classes).numel()) != B:
            raise ValueError(f"roi_classes has {torch.as_tensor(roi_classes).numel()} labels for {B} ROIs")
        groups = group_rois(roi_classes, self.members)
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32)
        if roi_cams.dim() == 2:
            roi_cams = roi_cams.unsqueeze(0).expand(B, 3, 3)
        inputs = dict(zip(_INPUTS, (f32(x), f32(roi_coord_2d), f32(roi_cams), f32(roi_centers), f32(roi_whs),
                                    f32(roi_extents), f32(resize_ratios).reshape(-1))))
        out = {"rot": torch.empty((B, 3, 3), dtype=torch.float32, device=dev),
               "trans": torch.empty((B, 3), dtype=torch.float32, device=dev)}
        if self.wants_maps:
            for name, ch in (("mask", 1), ("full_mask", 1), ("coor_x", 1), ("coor_y", 1), ("coor_z", 1), ("region", 65)):
                out[name] = torch.empty((B, ch, 64, 64), dtype=torch.float32, device=dev)
        if return_raw:
            out["raw"] = torch.empty((B, 9), dtype=torch.float32, device=dev)
        if B == 0:
            return out
        with torch.cuda.device(dev):
            caller = torch.cuda.current_stream()
            # a sub-batch above the member's max_batch runs eagerly (in chunks); capture before the fork, because
            # capture_graph synchronises the device
            graphed = {label: self.use_cuda_graph and idx.numel() <= self.members[label].max_batch for label, idx in groups}
            for label, idx in groups:
                if graphed[label]:
                    self._ensure_graph(label, idx, inputs, dev)
            fork = torch.cuda.Event()
            fork.record(caller)
            used = []
            for label, idx in groups:
                member, s = self.members[label], self._stream(label, dev)
                s.wait_event(fork)
                with torch.cuda.stream(s):
                    n = idx.numel()
                    idx_d = idx.to(dev, non_blocking=True)
                    if graphed[label]:
                        static, replay, o = self._graphs[(label, n)]
                        for k in _INPUTS:
                            torch.index_select(inputs[k], 0, idx_d, out=static[k])
                        replay()
                    else:
                        member._ensure_engine(dev)
                        ws = torch.empty(_lib.lib().gdrn_model_workspace_bytes(member._handle, min(n, member.max_batch)),
                                         dtype=torch.uint8, device=dev)
                        sub = {k: v.index_select(0, idx_d) for k, v in inputs.items()}
                        o = member(sub["roi_img"], roi_coord_2d=sub["roi_coord_2d"], roi_cams=sub["roi_cams"],
                                   roi_centers=sub["roi_centers"], roi_whs=sub["roi_whs"],
                                   roi_extents=sub["roi_extents"], resize_ratios=sub["resize_ratios"],
                                   return_raw=return_raw, _workspace=ws)
                    for k, t in out.items():
                        t.index_copy_(0, idx_d, o[k])
                # the caller's tensors are read / written on s: keep the allocator from recycling them before s is done
                for t in list(inputs.values()) + list(out.values()):
                    t.record_stream(s)
                used.append(s)
            for s in used:
                caller.wait_stream(s)
        return out

    def _ensure_graph(self, label, idx, inputs, dev):
        """Capture (once) the forward of ``label``'s member over static buffers of ``idx.numel()`` ROIs.  The buffers are
        first filled with this call's sub-batch, so the capture warm-up runs on real inputs."""
        key = (label, idx.numel())
        if key in self._graphs:
            return
        idx_d = idx.to(dev)
        static = {k: inputs[k].index_select(0, idx_d).contiguous() for k in _INPUTS}
        replay, o = self.members[label].capture_graph(static)
        self._graphs[key] = (static, replay, o)
