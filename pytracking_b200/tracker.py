"""Native whole-frame DiMP tracker behind the reference's tracker plug-in interface (`BaseTracker`:
pytracking/tracker/base/basetracker.py:6-22 -- `initialize(image, info) -> dict`, `track(image, info) -> {'target_bbox': [x,y,w,h]}`).

One `track()` = one C-ABI call (`b200trk_dimp_track_host`, include/b200trk.h): the uint8 frame goes to the GPU, the crop is sampled
there, backbone + head + classify + localisation run as kernels, 64 bytes come back, the float32 tracker state is advanced on the
host inside the library, and the online filter update is left running on the stream.  Nothing here falls back to PyTorch."""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .frame_engine import DiMPFrameEngine

FLAGS = {0: None, 1: "normal", 2: "hard_negative", 3: "uncertain", 4: "not_found"}

_DEFAULTS = dict(                                    # pytracking/parameter/dimp/dimp50.py + the `.get` defaults of dimp.py
    image_sample_size=288, search_area_scale=5, sample_memory_size=50, learning_rate=0.01, hard_negative_learning_rate=None,
    init_samples_minimum_weight=None, train_skipping=1, train_sample_interval=1, net_opt_iter=None, net_opt_update_iter=None,
    net_opt_hn_iter=None, update_classifier=False, advanced_localization=False, target_not_found_threshold=0.0,
    distractor_threshold=0.0, hard_negative_threshold=0.0, target_neighborhood_scale=0.0, dispalcement_scale=0.0,
    uncertain_threshold=-math.inf, hard_sample_threshold=-math.inf, target_inside_ratio=0.2, augmentation_expansion_factor=None,
    output_not_found_box=False, use_iou_net=True, iounet_k=5, num_init_random_boxes=0, box_jitter_pos=0.0, box_jitter_sz=0.0,
    maximal_aspect_ratio=6.0, box_refinement_iter=0, box_refinement_step_length=1.0, box_refinement_step_decay=1.0,
    box_refinement_space="default", update_scale_when_uncertain=True, use_iounet_pos_for_learning=True,
    border_mode="replicate", patch_max_scale_change=None, score_preprocess="none", softmax_reg=None, score_filter_ksz=1,
    low_score_opt_threshold=None)

BORDER_MODES = {"replicate": 0, "inside": 1, "inside_major": 2}
SCORE_PREPROCESS = {"none": 0, "exp": 1, "softmax": 2}

# PrDiMPSteepestDescentNewton's constructor arguments (ltr/models/target_classifier/optimizer.py:312-314) with its defaults
NEWTON_DEFAULTS = dict(feat_stride=16, init_step_length=1.0, init_filter_reg=1e-2, gauss_sigma=1.0, min_filter_reg=1e-3, alpha_eps=0.0,
                       init_uni_weight=None, normalize_label=False, label_shrink=0, softmax_reg=None, label_threshold=0.0)
# TrackerParams entries that DiMP._overwrite_classifier_params (dimp.py:589-603) writes into the filter optimiser
_NEWTON_PARAM_OVERRIDES = ("filter_reg", "softmax_reg", "label_threshold", "label_shrink")


def newton_hparams(newton, params_source=None, **param_overrides):
    """The Newton optimiser's hyper-parameters (constructor names; `init_step_length` / `init_filter_reg` stand for the learnt
    exp(log_step_length) / filter_reg) after the TrackerParams overrides of _overwrite_classifier_params: params.filter_reg sets both
    filter_reg and min_filter_reg (and is recorded as `filter_reg_override`, which takes precedence over a learnt filter_reg in the
    state_dict); softmax_reg, label_threshold and label_shrink replace the optimiser's own values."""
    unknown = set(newton) - set(NEWTON_DEFAULTS) - {"filter_reg_override"}
    if unknown:
        raise ValueError("b200trk: unknown PrDiMPSteepestDescentNewton arguments %s" % sorted(unknown))
    h = dict(NEWTON_DEFAULTS, **newton)
    for k in _NEWTON_PARAM_OVERRIDES:
        v = param_overrides.get(k, getattr(params_source, k, None) if params_source is not None else None)
        if v is None:
            continue
        if k == "filter_reg":          # pred_module.filter_reg[0] = min_filter_reg = params.filter_reg, whatever the net had learnt
            h["init_filter_reg"] = h["min_filter_reg"] = h["filter_reg_override"] = float(v)
        else:
            h[k] = v
    return h


def make_params(source=None, **overrides):
    """b200trk_dimp_params_t from a reference `TrackerParams` object (attribute access) and / or keyword overrides."""
    vals = dict(_DEFAULTS)
    if source is not None:
        for k in vals:
            if hasattr(source, k):
                vals[k] = getattr(source, k)
    vals.update(overrides)
    p = _lib.DimpParams()
    none_int = lambda v: -1 if v is None else int(v)
    p.image_sample_size = int(vals["image_sample_size"])
    p.search_area_scale = float(vals["search_area_scale"])
    p.sample_memory_size = int(vals["sample_memory_size"])
    p.learning_rate = float(vals["learning_rate"])
    p.hard_negative_learning_rate = -1.0 if vals["hard_negative_learning_rate"] is None else float(vals["hard_negative_learning_rate"])
    p.init_samples_minimum_weight = float(vals["init_samples_minimum_weight"] or 0.0)
    p.train_skipping, p.train_sample_interval = int(vals["train_skipping"]), int(vals["train_sample_interval"])
    p.net_opt_iter, p.net_opt_update_iter = none_int(vals["net_opt_iter"]), none_int(vals["net_opt_update_iter"])
    p.net_opt_hn_iter = none_int(vals["net_opt_hn_iter"])
    p.update_classifier, p.advanced_localization = int(bool(vals["update_classifier"])), int(bool(vals["advanced_localization"]))
    for k in ("target_not_found_threshold", "distractor_threshold", "hard_negative_threshold", "target_neighborhood_scale",
              "dispalcement_scale", "uncertain_threshold", "hard_sample_threshold", "target_inside_ratio"):
        setattr(p, k, float(vals[k]))
    p.augmentation_expansion_factor = float(vals["augmentation_expansion_factor"] or 0.0)
    p.output_not_found_box = int(bool(vals["output_not_found_box"]))
    p.use_iou_net, p.iounet_k = int(bool(vals["use_iou_net"])), int(vals["iounet_k"])
    p.num_init_random_boxes = int(vals["num_init_random_boxes"])
    p.box_jitter_pos, p.box_jitter_sz = float(vals["box_jitter_pos"]), float(vals["box_jitter_sz"])
    p.maximal_aspect_ratio = float(vals["maximal_aspect_ratio"])
    p.box_refinement_iter = int(vals["box_refinement_iter"])
    if isinstance(vals["box_refinement_step_length"], (tuple, list)):
        raise NotImplementedError("b200trk: per-coordinate box_refinement_step_length")
    p.box_refinement_step_length, p.box_refinement_step_decay = float(vals["box_refinement_step_length"]), float(vals["box_refinement_step_decay"])
    p.box_refinement_relative = int(vals["box_refinement_space"] == "relative")
    p.update_scale_when_uncertain = int(bool(vals["update_scale_when_uncertain"]))
    p.use_iounet_pos_for_learning = int(bool(vals["use_iounet_pos_for_learning"]))
    if vals["border_mode"] not in BORDER_MODES:
        raise NotImplementedError("b200trk: border_mode %r (supported: %s)" % (vals["border_mode"], ", ".join(BORDER_MODES)))
    p.border_mode = BORDER_MODES[vals["border_mode"]]
    p.patch_max_scale_change = 0.0 if vals["patch_max_scale_change"] is None else float(vals["patch_max_scale_change"])
    if vals["score_preprocess"] not in SCORE_PREPROCESS:
        raise NotImplementedError("b200trk: score_preprocess %r (supported: %s)" % (vals["score_preprocess"], ", ".join(SCORE_PREPROCESS)))
    p.score_preprocess = SCORE_PREPROCESS[vals["score_preprocess"]]
    p.has_softmax_reg = int(vals["softmax_reg"] is not None)
    p.softmax_reg = 0.0 if vals["softmax_reg"] is None else float(vals["softmax_reg"])
    if int(vals["score_filter_ksz"]) > 1:
        raise NotImplementedError("b200trk: score_filter_ksz > 1 (a box filter on the score map) is not implemented")
    if vals["low_score_opt_threshold"] is not None:
        raise NotImplementedError("b200trk: low_score_opt_threshold (net_opt_low_iter schedule) is not implemented")
    return p


def tracker_settings(params, newton, **param_overrides):
    """(b200trk_dimp_params_t, Newton hyper-parameters or None) of a tracker.  `params`: a DimpParams, used as it is, or a
    `TrackerParams` source for make_params.  For PrDiMP (`newton` a dict) the params' filter_reg / softmax_reg / label_threshold /
    label_shrink apply to the optimiser (newton_hparams), and the localisation's softmax uses the optimiser's softmax_reg, as
    localize_target does (dimp.py:207)."""
    own = isinstance(params, _lib.DimpParams)
    p = params if own else make_params(params, **param_overrides)
    if newton is not None:
        newton = newton_hparams(newton, None if own else params, **param_overrides)
        p.has_softmax_reg = int(newton["softmax_reg"] is not None)
        p.softmax_reg = 0.0 if newton["softmax_reg"] is None else float(newton["softmax_reg"])
    return p, newton


def augmentation_from_params(tp):
    """(augmentation, random_shift_factor) for DiMPTracker from a reference `TrackerParams`: params.augmentation when
    use_augmentation is set (absent means set, as generate_init_samples reads it), else (None, 0.0) -- the un-augmented start."""
    if not getattr(tp, "use_augmentation", True) or getattr(tp, "augmentation", None) is None:
        return None, 0.0
    return dict(tp.augmentation), float(getattr(tp, "random_shift_factor", 0) or 0)


def augmentation_samples(augmentation):
    """First-frame samples an augmentation dict gives: the identity, its transforms and its dropout copies."""
    a = augmentation
    if "scale" in a:
        raise NotImplementedError("b200trk: augmentation 'scale' is not implemented (no DiMP-family parameter file uses it)")
    return (1 + len(a.get("shift", [])) + len(a.get("relativeshift", [])) + int(bool(a.get("fliplr"))) + len(a.get("blur", [])) +
            len(a.get("rotate", [])) + int(a.get("dropout", (0, 0))[0]))


def draw_augmentation(augmentation, image_sample_size, random_shift_factor, feature_dim):
    """The b200trk_dimp_augment_t of one augmented initialisation, with every random number drawn as the reference draws it
    (generate_init_samples, dimp.py:364-388, then init_classifier's dropout, dimp.py:544-547) from torch's CPU generator: the flip,
    blur and rotate shifts in that order, then F.dropout2d's masks -- drawn on ones [num, C, 1, 1], which consumes the generator
    exactly as dropout2d on the features does.  -> (descriptor, multipliers tensor kept alive by the caller)."""
    a = augmentation
    augmentation_samples(a)
    iss = torch.Tensor([image_sample_size, image_sample_size])
    if random_shift_factor > 0:
        rand_shift = lambda: ((torch.rand(2) - 0.5) * iss * random_shift_factor).long().tolist()
    else:
        rand_shift = lambda: [0, 0]
    K = _lib.AUG_KINDS
    xf = [(K["identity"], [0, 0], (0.0, 0.0))]
    xf += [(K["translation"], [int(s[0]), int(s[1])], (0.0, 0.0)) for s in a.get("shift", [])]
    xf += [(K["translation"], (torch.Tensor(s) * iss / 2).long().tolist(), (0.0, 0.0)) for s in a.get("relativeshift", [])]
    if a.get("fliplr"):
        xf.append((K["fliplr"], rand_shift(), (0.0, 0.0)))
    for sg in a.get("blur", []):
        xf.append((K["blur"], rand_shift(), tuple(float(v) for v in (sg if isinstance(sg, (tuple, list)) else (sg, sg)))))
    for ang in a.get("rotate", []):
        xf.append((K["rotate"], rand_shift(), (float(ang), 0.0)))
    num, prob = a.get("dropout", (0, 0.0))
    d = _lib.DimpAugment()
    d.num_transforms = len(xf)
    for k, (kind, shift, param) in enumerate(xf):
        d.transform[k].kind, d.transform[k].shift[0], d.transform[k].shift[1] = kind, int(shift[0]), int(shift[1])
        d.transform[k].param[0], d.transform[k].param[1] = param
    mult = None
    if int(num) > 0:
        mult = torch.nn.functional.dropout2d(torch.ones(int(num), feature_dim, 1, 1), p=prob, training=True).reshape(int(num), -1).contiguous()
        d.num_dropout, d.dropout_mult = int(num), mult.data_ptr()
    return d, mult


def frame_pointer(image, staging, key, who):
    """A uint8 [H,W,3] RGB frame -> (keep-alive, pointer, H, W, on_device).  A CUDA tensor or a pinned host tensor is used in place.
    Any other frame (ndarray, pageable tensor) is copied into the pinned buffer staging[key], which is reused while the frame size
    stays the same; the library then uploads it with one asynchronous copy."""
    if isinstance(image, torch.Tensor) and (image.is_cuda or image.is_pinned()):
        if image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3 or not image.is_contiguous():
            raise RuntimeError("%s: a frame tensor must be contiguous uint8 [H,W,3], got %s %s" % (who, image.dtype, tuple(image.shape)))
        return image, image.data_ptr(), int(image.shape[0]), int(image.shape[1]), image.is_cuda
    a = np.ascontiguousarray(image)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
        raise RuntimeError("%s: a frame must be uint8 [H,W,3] (RGB), got %s %s" % (who, a.dtype, a.shape))
    buf = staging.get(key)
    if buf is None or tuple(buf.shape) != a.shape:
        buf = staging[key] = torch.empty(a.shape, dtype=torch.uint8).pin_memory()
    buf.numpy()[...] = a
    return buf, buf.data_ptr(), a.shape[0], a.shape[1], False


class HostLogic:
    """The host half of the tracker alone (no GPU): crop planning and the post-localisation state update.  Used by the CPU tests."""

    def __init__(self, params):
        self.params = params
        h = C.c_void_p()
        _lib.check(_lib.lib().b200trk_dimp_tracker_create(C.byref(h), None, C.byref(params)), "dimp_tracker_create")
        self.handle = h

    def init_state(self, H, W, init_bbox):
        g, box = _lib.CropGeom(), (C.c_float * 4)()
        bb = (C.c_double * 4)(*[float(v) for v in init_bbox])
        _lib.check(_lib.lib().b200trk_dimp_tracker_init_state(self.handle, H, W, C.byref(bb), C.byref(g), C.byref(box)), "init_state")
        return g, np.array(box, dtype=np.float32)

    def init_state_augmented(self, H, W, init_bbox, augment):
        """Host half of the augmented initialize for a drawn descriptor (draw_augmentation) -> (crop geometry, target boxes [n,4])."""
        n = augment.num_transforms + augment.num_dropout
        g, boxes = _lib.CropGeom(), np.zeros((max(n, 1), 4), np.float32)
        bb = (C.c_double * 4)(*[float(v) for v in init_bbox])
        _lib.check(_lib.lib().b200trk_dimp_tracker_init_state_augmented(self.handle, H, W, C.byref(bb), C.byref(augment), C.byref(g),
                                                                        boxes.ctypes.data_as(C.c_void_p)), "init_state_augmented")
        return g, boxes[:n]

    def adopt(self, H, W, state9, sample_weights, num_stored, num_init, previous_replace_ind=-1, frame_num=1):
        s = [float(v) for v in state9]
        sw = np.ascontiguousarray(sample_weights, dtype=np.float32)
        _lib.check(_lib.lib().b200trk_dimp_tracker_adopt(
            self.handle, H, W, C.byref((C.c_float * 2)(s[0], s[1])), C.byref((C.c_float * 2)(s[2], s[3])), s[4],
            C.byref((C.c_float * 2)(s[5], s[6])), s[7], s[8], sw.ctypes.data_as(C.c_void_p), int(num_stored), int(num_init),
            int(previous_replace_ind), int(frame_num)), "adopt")

    def plan_crop(self):
        g = _lib.CropGeom()
        _lib.check(_lib.lib().b200trk_dimp_tracker_plan_crop(self.handle, C.byref(g)), "plan_crop")
        return g

    def commit(self, geom, loc):
        info = _lib.FrameInfo()
        sw = np.zeros(self.params.sample_memory_size, dtype=np.float32)
        _lib.check(_lib.lib().b200trk_dimp_tracker_commit(self.handle, C.byref(geom), C.byref(loc), C.byref(info),
                                                          sw.ctypes.data_as(C.c_void_p)), "commit")
        return info, sw

    def state(self):
        out = (C.c_float * 9)()
        _lib.check(_lib.lib().b200trk_dimp_tracker_state(self.handle, C.byref(out)), "state")
        return np.array(out, dtype=np.float32)

    def close(self):
        if getattr(self, "handle", None):
            _lib.lib().b200trk_dimp_tracker_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DiMPTracker(HostLogic):
    """initialize / track on one GPU.  `state_dict`: the DiMP network's state_dict (reference key names).
    `newton`: None for DiMP; for PrDiMP the PrDiMPSteepestDescentNewton constructor arguments (NEWTON_DEFAULTS names), to which
    params.filter_reg / softmax_reg / label_threshold / label_shrink apply as in DiMP._overwrite_classifier_params.  The localisation's
    softmax then uses the optimiser's softmax_reg, as localize_target does (dimp.py:207).
    `filter_init`: the filter `initialize` starts the optimiser from -- "zero" (FilterInitializerZero, the reference under
    filter_init_zero) or "network" (the network's FilterInitializerLinear, the reference otherwise; `init_filter_norm` /
    `init_pool_square` are its constructor arguments, False in dimpnet50 and klcedimpnet50).
    `augmentation`: None starts from the un-augmented first-frame sample; a dict in the form of the reference's params.augmentation
    (with `random_shift_factor`, see augmentation_from_params) starts as DiMP.initialize does with use_augmentation: the transformed
    crops, the dropout copies and a first optimisation over all of them.  The network is then sized for that many samples."""

    def __init__(self, state_dict, params=None, arch="resnet50", precision=0, device=None, newton=None, filter_init="zero",
                 init_filter_norm=False, init_pool_square=False, augmentation=None, random_shift_factor=0.0, **param_overrides):
        self.params, newton = tracker_settings(params, newton, **param_overrides)
        p = self.params
        self.augmentation = None if augmentation is None else dict(augmentation)
        self.random_shift_factor = float(random_shift_factor or 0.0)
        n = 1 if self.augmentation is None else augmentation_samples(self.augmentation)
        if n > _lib.AUG_MAX:
            raise ValueError("DiMPTracker: the augmentation gives %d first-frame samples (at most %d)" % (n, _lib.AUG_MAX))
        self.engine = DiMPFrameEngine(state_dict, arch=arch, filter_size=4, memory_size=p.sample_memory_size, max_batch=n,
                                      crop_size=p.image_sample_size, precision=precision, device=device, newton=newton,
                                      filter_init=filter_init, init_filter_norm=init_filter_norm, init_pool_square=init_pool_square)
        self.device = self.engine.device
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_dimp_tracker_create(C.byref(h), self.engine.state, C.byref(p)), "dimp_tracker_create")
        self.handle = h
        self.info = _lib.FrameInfo()
        self.debug_info = {}
        self._pinned = {}
        self.iou = None
        self.torch_noise = False       # True: draw the random proposals' noise with torch.rand, exactly where the reference does

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _frame(self, image, on_device):
        keep, ptr, H, W, dev = frame_pointer(image, self._pinned, 0, "DiMPTracker")
        if dev != on_device:
            raise RuntimeError("DiMPTracker: this call takes a frame %s" % ("on the GPU" if on_device else "on the host"))
        return keep, ptr, H, W

    def initialize(self, image, info):
        """DiMP.initialize: un-augmented (b200trk_dimp_tracker_initialize_host), or with the tracker's augmentation, whose random
        numbers come from torch's CPU generator in the reference's order (draw_augmentation;
        b200trk_dimp_tracker_initialize_augmented_host)."""
        keep, ptr, H, W = self._frame(image, False)
        bb = (C.c_double * 4)(*[float(v) for v in info["init_bbox"]])
        L = _lib.lib()
        with torch.cuda.device(self.device):
            if self.augmentation is None:
                _lib.check(L.b200trk_dimp_tracker_initialize_host(self.handle, C.c_void_p(ptr), H, W, C.byref(bb), self._stream()),
                           "dimp_tracker_initialize_host")
            else:
                d, mult = draw_augmentation(self.augmentation, self.params.image_sample_size, self.random_shift_factor,
                                            self.engine.feat_dims[0])
                _lib.check(L.b200trk_dimp_tracker_initialize_augmented_host(self.handle, C.c_void_p(ptr), H, W, C.byref(bb), C.byref(d),
                                                                            self._stream()), "dimp_tracker_initialize_augmented_host")
        return {}

    def attach_iounet(self, state_dict, modulation=None):
        """IoUNet refinement: `state_dict` of the whole DiMP network (bb_regressor.* keys).  `modulation`: the two modulation vectors
        of the first-frame target (AtomIoUNet.get_modulation; DiMP.init_iou_net dimp.py:509-540), or None to compute them natively
        from the bb_regressor's conv3_1r / conv4_1r / fc3_1r / fc34_*r weights during `initialize` (attach before it)."""
        from .iou import IoUModulation, IoUPredictor
        bb = self.engine.backbone
        if not getattr(bb, "iou_dims", None):
            bb.attach_iou_head(state_dict)
        L = _lib.lib()
        with torch.cuda.device(self.device):
            if modulation is None:
                if not getattr(bb, "has_iou_ref", False):
                    bb.attach_iou_ref(state_dict)
                head = IoUModulation(state_dict, device=self.device)
                _lib.check(L.b200trk_dimp_tracker_attach_modulation_head(self.handle, head.handle), "dimp_tracker_attach_modulation_head")
                self.modulation_head = head            # the library holds the handle from here on
                m3 = m4 = None
            else:
                m3 = modulation[0].detach().float().reshape(-1).cpu().contiguous()
                m4 = modulation[1].detach().float().reshape(-1).cpu().contiguous()
            pred = IoUPredictor(state_dict, device=self.device)
            _lib.check(L.b200trk_dimp_tracker_attach_iounet(self.handle, pred.handle, None if m3 is None else C.c_void_p(m3.data_ptr()),
                                                            None if m4 is None else C.c_void_p(m4.data_ptr())), "dimp_tracker_attach_iounet")
            self.iou = pred

    def modulation(self):
        """(mod3, mod4) float32 numpy: the modulation vectors the IoUNet uses."""
        m3, m4 = np.zeros(self.iou.C3, np.float32), np.zeros(self.iou.C4, np.float32)
        _lib.check(_lib.lib().b200trk_dimp_tracker_modulation(self.handle, m3.ctypes.data_as(C.c_void_p), m4.ctypes.data_as(C.c_void_p)),
                   "dimp_tracker_modulation")
        return m3, m4

    @staticmethod
    def newton_from_reference(ref):
        """PrDiMPSteepestDescentNewton hyper-parameters of a reference PrDiMP `DiMP` object (after its initialize(), i.e. with the
        parameter overrides already written into the optimiser), in the constructor's names."""
        fo = ref.net.classifier.filter_optimizer
        return dict(feat_stride=fo.feat_stride, init_step_length=float(torch.exp(fo.log_step_length.detach().float()).item()),
                    init_filter_reg=float(fo.filter_reg.detach().float().reshape(-1)[0].item()), gauss_sigma=fo.gauss_sigma,
                    min_filter_reg=fo.min_filter_reg, alpha_eps=fo.alpha_eps, init_uni_weight=fo.uni_weight,
                    normalize_label=fo.normalize_label, label_shrink=fo.label_shrink, softmax_reg=fo.softmax_reg,
                    label_threshold=fo.label_threshold)

    def adopt_reference(self, ref, image_hw):
        """Take over from a reference `DiMP` or PrDiMP `DiMP` object after its `initialize()` (any augmentation / initialiser):
        scalars, sample weights, sample memory, boxes and filter are copied into the engine; tracking continues natively.  For PrDiMP
        the engine must have been built with the Newton optimiser (`newton=DiMPTracker.newton_from_reference(ref)`)."""
        e = self.engine
        is_newton = type(ref.net.classifier.filter_optimizer).__name__ == "PrDiMPSteepestDescentNewton"
        if is_newton != (e.newton is not None):
            raise RuntimeError("DiMPTracker.adopt_reference: the reference runs %s, this tracker's state %s" % (
                type(ref.net.classifier.filter_optimizer).__name__, "PrDiMPSteepestDescentNewton" if e.newton else "DiMPSteepestDescentGN"))
        if is_newton:
            nw = self.newton_from_reference(ref)
            mine = {k: e.newton[k] for k in nw}
            if any(float(nw[k] or 0) != float(mine[k] or 0) for k in nw if k not in ("init_step_length", "init_filter_reg")) or \
                    (nw["softmax_reg"] is None) != (mine["softmax_reg"] is None):
                raise RuntimeError("DiMPTracker.adopt_reference: Newton hyper-parameters differ from the reference's: %s vs %s" % (mine, nw))
        n = int(min(int(ref.num_stored_samples[0]), self.params.sample_memory_size))
        e.memory[:n].copy_(ref.training_samples[0][:n].to(self.device))
        e.boxes[:n].copy_(ref.target_boxes[:n].to(self.device))
        e.sample_weights.copy_(ref.sample_weights[0].to(self.device))
        e.filter.copy_(ref.target_filter.reshape(e.filter.shape).to(self.device))
        st = [float(ref.pos[0]), float(ref.pos[1]), float(ref.target_sz[0]), float(ref.target_sz[1]), float(ref.target_scale),
              float(ref.base_target_sz[0]), float(ref.base_target_sz[1]), float(ref.min_scale_factor), float(ref.max_scale_factor)]
        prev = ref.previous_replace_ind[0]
        self.adopt(int(image_hw[0]), int(image_hw[1]), st, ref.sample_weights[0].detach().float().cpu().numpy(),
                   int(ref.num_stored_samples[0]), int(ref.num_init_samples[0]), -1 if prev is None else int(prev), int(ref.frame_num))
        if self.params.use_iou_net and self.iou is None:
            self.attach_iounet(ref.net.net.state_dict(), ref.iou_modulation)
        torch.cuda.synchronize(self.device)

    def _noise(self):
        n = self.params.num_init_random_boxes
        if self.torch_noise and self.params.use_iou_net and n > 0:
            u = torch.rand(n, 4).contiguous()                          # dimp.py:667
            _lib.check(_lib.lib().b200trk_dimp_tracker_set_proposal_noise(self.handle, C.c_void_p(u.data_ptr()), 4 * n), "set_proposal_noise")

    def track(self, image, info=None):
        self._noise()
        keep, ptr, H, W = self._frame(image, False)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_dimp_track_host(self.handle, C.c_void_p(ptr), H, W, C.byref(self.info), self._stream()),
                       "dimp_track_host")
        self.debug_info = {"flag": FLAGS[self.info.flag], "max_score": float(self.info.max_score),
                           "predicted_iou": float(self.info.predicted_iou) if self.info.refined else None}
        return {"target_bbox": [float(v) for v in self.info.bbox]}

    def track_device(self, image_dev):
        """`track` with the uint8 [H,W,3] frame already on the GPU (a CUDA tensor)."""
        self._noise()
        keep, ptr, H, W = self._frame(image_dev, True)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_dimp_track_device(self.handle, C.c_void_p(ptr), H, W, C.byref(self.info), self._stream()),
                       "dimp_track_device")
        return self.info

    def close(self):
        HostLogic.close(self)
        if getattr(self, "iou", None) is not None:
            self.iou.close()
            self.iou = None
        if getattr(self, "modulation_head", None) is not None:
            self.modulation_head.close()
            self.modulation_head = None
        if getattr(self, "engine", None) is not None:
            self.engine.close()
            self.engine = None
