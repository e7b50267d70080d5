"""Host-side mirror of the reference's plug-in seams for the hot path (SURVEY.md 8(b)) -- same names, argument meaning,
return contracts and shape conventions as the reference functions / modules they stand in for, computing through the
C-ABI library.  `install()` rebinds the seams inside an importable, unmodified pytracking checkout (INTEGRATION.md).

Shapes the CUDA path does not claim (several sequences per call, filter sizes other than 4x4, dilation, groups,
training mode) raise `NotImplementedError` here; `install()` keeps the reference implementation for exactly those cases.

Each section below serves one reference module: its mirrors and the served paths that call them.  A seam `seam(reference, *args,
**kwargs)` receives the implementation it replaces and hands the call to `_serve`; `SEAMS` at the end lists what `install()` binds,
building each seam of one served path with `_seam` (the seams that try several served paths are written out beside them).
"""
import contextlib
import functools
import importlib
import os
import time
import weakref

import torch

from . import eco_plan, ops
from .engine import BackboneEngine
from .iou import IoUPredictor
from .transformer_engine import BoxTower, TokenBuilder, TransformerEngine


# ---------------------------------------------------------------------------------------------------------------
# the fall-through rule, call accounting and the state of one install()
# ---------------------------------------------------------------------------------------------------------------
stats = {}               # seam name -> number of calls served by the CUDA library (tests / bench read this)
seam_seconds = {}        # seam name -> device-synchronised seconds spent inside the library call (only with B200TRK_PLUGIN_TIMING=1)
_TIMING = bool(int(os.environ.get("B200TRK_PLUGIN_TIMING", "0")))


def _count(name):
    stats[name] = stats.get(name, 0) + 1


def _serve(name, served, reference, *args, **kwargs):
    """`served` raises NotImplementedError for a call the CUDA path does not claim, before it touches the library or the caller's
    objects; that call goes to `reference` with exactly the caller's arguments.  A call `served` returns from counts under `name`."""
    try:
        out = served(*args, **kwargs)
    except NotImplementedError:
        return reference(*args, **kwargs)
    _count(name)
    return out


def _seam(name, served):
    """The seam `seam(reference, *args, **kwargs)` of a single served path."""
    return functools.partial(_serve, name, served)


@contextlib.contextmanager
def _timed(name):
    """with _timed(name): ... -- wall time of the block with a device synchronisation on both sides (debugging aid, off by default)."""
    if not _TIMING:
        yield
        return
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        yield
    finally:
        torch.cuda.synchronize()
        seam_seconds[name] = seam_seconds.get(name, 0.0) + time.perf_counter() - t0


def _inference(*tensors):
    """The CUDA path serves inference calls only: CUDA fp32 tensors, nothing that autograd has to differentiate."""
    for t in tensors:
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
            return False
        if torch.is_grad_enabled() and t.requires_grad:
            return False
    return True


class _State:
    """Engines, mirror objects and caches of one `install()`, keyed weakly on the reference's modules; `uninstall()` drops it."""

    def __init__(self, max_batch, precision):
        self.max_batch, self.precision = max_batch, precision
        self.engines = weakref.WeakKeyDictionary()       # net module -> {(H, W): BackboneEngine}
        self.last_pass = weakref.WeakKeyDictionary()     # net module -> (engine, [layer2, layer3] tensors it returned, batch) of the last pass
        self.mirrors = weakref.WeakKeyDictionary()       # optimiser module -> (its parameter versions and settings, mirror object)
        self.towers = weakref.WeakKeyDictionary()        # DenseBoxRegressor -> {(H, W): BoxTower}
        self.builders = weakref.WeakKeyDictionary()      # FilterPredictor -> {"builder": TokenBuilder, "const": {shape key: (pos, mask)}}
        self.predictors = weakref.WeakKeyDictionary()    # AtomIoUNet -> IoUPredictor
        self.tr_engines = weakref.WeakKeyDictionary()    # Transformer -> {(tokens, batch): TransformerEngine}
        self.head_cache = weakref.WeakKeyDictionary()    # Head -> {(data_ptr, shape, version): feature}


_state = None


# ---------------------------------------------------------------------------------------------------------------
# ltr/models/layers/filter.py
# ---------------------------------------------------------------------------------------------------------------
_CORR_SLOTS = {18: 16, 22: 8}        # channel granularity of the correlation kernels per feature size (csrc/corr.cuh CorrSlots)


def _check_corr_shape(f, who):
    """Everything the C library would reject (corr_api.cu / sd_optimizer.cu argument checks) is rejected here with
    NotImplementedError, so that `install()` can keep the reference implementation for exactly those calls."""
    if f.dim() != 4 or f.dtype != torch.float32:
        raise NotImplementedError("b200trk %s: float32 [n,C,H,W] features" % who)
    h, w, c = f.shape[-2], f.shape[-1], f.shape[-3]
    if h != w or h not in _CORR_SLOTS or c % _CORR_SLOTS[h] != 0 or f.shape[0] < 1 or f.shape[0] > 1024:
        raise NotImplementedError("b200trk %s: feature maps of 18x18 or 22x22 with C a multiple of 16 / 8 (got %s)" % (who, tuple(f.shape)))


def apply_filter(feat, filter, dilation_factors=None):
    """filter.py:5-57. feat (images_in_sequence, [sequences], feat_dim, H, W); filter (sequences, feat_dim, fH, fW)
    -> scores (images_in_sequence, [sequences], yH, yW)."""
    multiple_filters = (filter.dim() == 5)
    if dilation_factors is not None or multiple_filters:
        raise NotImplementedError("b200trk apply_filter: dilation / multiple filters are not on the CUDA path")
    num_images = feat.shape[0]
    num_sequences = feat.shape[1] if feat.dim() == 5 else 1
    if num_sequences != 1 or filter.shape[0] != 1:
        raise NotImplementedError("b200trk apply_filter: one sequence per call")
    f = feat.reshape(num_images, *feat.shape[-3:])
    if filter.shape[-1] == 1 and filter.shape[-2] == 1:
        # _apply_filter_ksz1 (filter.py:60-88, the ToMP classifier): a matmul over the channels == a 1x1 convolution
        scores = ops.conv1x1(f, filter.reshape(1, filter.shape[-3], 1, 1))
        return scores.reshape(num_images, num_sequences, scores.shape[-2], scores.shape[-1])
    if filter.shape[-1] != 4 or filter.shape[-2] != 4:
        raise NotImplementedError("b200trk apply_filter: 4x4 or 1x1 filters")
    _check_corr_shape(f, "apply_filter")
    scores = ops.apply_filter(f, filter.reshape(1, *filter.shape[-3:]))
    return scores.reshape(num_images, num_sequences, scores.shape[-2], scores.shape[-1])


def apply_feat_transpose(feat, input, filter_ksz, training=True, groups=1):
    """filter.py:91-107 (v2 and v3 are the same adjoint). input (images, [sequences], yH, yW) -> (sequences, feat_dim, fH, fW)."""
    if groups != 1:
        raise NotImplementedError("b200trk apply_feat_transpose: groups != 1")
    if isinstance(filter_ksz, int):
        filter_ksz = (filter_ksz, filter_ksz)
    num_images = feat.shape[0]
    num_sequences = feat.shape[1] if feat.dim() == 5 else 1
    if num_sequences != 1 or tuple(filter_ksz) != (4, 4):
        raise NotImplementedError("b200trk apply_feat_transpose: one sequence and a 4x4 filter per call")
    f = feat.reshape(num_images, *feat.shape[-3:])
    _check_corr_shape(f, "apply_feat_transpose")
    r = input.reshape(num_images, 1, input.shape[-2], input.shape[-1])
    return ops.apply_feat_transpose(f, r, 4)


def _served_apply_filter(feat, filter, dilation_factors=None):
    if not _inference(feat, filter):
        raise NotImplementedError("b200trk apply_filter: CUDA float32 tensors outside autograd")
    return apply_filter(feat, filter, dilation_factors)


def _served_apply_feat_transpose(feat, input, filter_ksz, training=True, groups=1):
    if not _inference(feat, input):
        raise NotImplementedError("b200trk apply_feat_transpose: CUDA float32 tensors outside autograd")
    return apply_feat_transpose(feat, input, filter_ksz, training, groups)


# ---------------------------------------------------------------------------------------------------------------
# pytracking/libs/dcf.py, pytracking/libs/operation.py (ATOM)
# ---------------------------------------------------------------------------------------------------------------
def max2d(a):
    """dcf.py:156-164 -> (max_val, argmax [.., 2] as (row, col))."""
    return ops.max2d(a)


def _served_max2d(a):
    if not (_inference(a) and a.dim() >= 2):
        raise NotImplementedError("b200trk max2d: a CUDA float32 tensor of at least two dimensions")
    return max2d(a)


def _plain_conv(input, weight, bias, stride, padding, dilation, groups):
    if not (weight is not None and _inference(input, weight) and input.dim() == 4 and weight.dim() == 4 and bias is None and
            stride == 1 and padding == 0 and dilation == 1 and groups == 1):
        raise NotImplementedError("b200trk operation.conv2d: 4-D CUDA float32 operands without bias, stride, padding, dilation or groups")


def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1, mode=None):
    """operation.py:5-32 for ATOM.apply_filter: one 4x4 filter, mode='same'."""
    _plain_conv(input, weight, bias, stride, padding, dilation, groups)
    if not (mode == "same" and weight.shape[0] == 1 and weight.shape[2] == 4 and weight.shape[3] == 4):
        raise NotImplementedError("b200trk conv2d: only mode='same' with a single 4x4 filter is on the CUDA path")
    _check_corr_shape(input, "conv2d")
    return ops.conv2d_same(input, weight)


def conv1x1(input, weight):
    """operation.py:35-42."""
    if not (weight is not None and _inference(input, weight) and input.dim() == 4 and weight.dim() == 4 and weight.shape[2] == 1 and
            weight.shape[3] == 1):
        raise NotImplementedError("b200trk conv1x1: 4-D CUDA float32 operands with a 1x1 filter")
    return ops.conv1x1(input, weight)


def _conv2d_as_conv1x1(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1, mode=None):
    """operation.conv2d with a 1x1 filter and no padding mode (ATOM's feature projection) is conv1x1."""
    _plain_conv(input, weight, bias, stride, padding, dilation, groups)
    if not (mode is None and weight.shape[2] == 1 and weight.shape[3] == 1 and input.shape[1] == weight.shape[1] and
            input.shape[-1] * input.shape[-2] > 1):
        raise NotImplementedError("b200trk operation.conv2d: a 1x1 filter over all input channels, no mode")
    return conv1x1(input, weight)


def operation_conv2d(reference, *args, **kwargs):
    """ATOM's filter ('same', one 4x4 filter), else its 1x1 projection, else the reference; each served path counts by its name."""
    as_conv1x1 = functools.partial(_serve, "operation.conv1x1", _conv2d_as_conv1x1, reference)
    return _serve("operation.conv2d", conv2d, as_conv1x1, *args, **kwargs)


# ---------------------------------------------------------------------------------------------------------------
# ltr/models/target_classifier/optimizer.py  (forward(weights, feat, bb, sample_weight, num_iter, compute_losses)
#                                            -> (weights, weight_iterates, losses))
# ---------------------------------------------------------------------------------------------------------------
def _one_sequence(feat, bb, sample_weight):
    num_images = feat.shape[0]
    num_sequences = feat.shape[1] if feat.dim() == 5 else 1
    if num_sequences != 1:
        raise NotImplementedError("b200trk optimiser modules: one sequence per call (the tracker's inference configuration)")
    f = feat.reshape(num_images, *feat.shape[-3:])
    _check_corr_shape(f, "optimiser module")
    b = None if bb is None else bb.reshape(num_images, 4).float()
    sw = None
    if isinstance(sample_weight, torch.Tensor):
        sw = sample_weight.reshape(num_images).float()
    elif sample_weight is not None:
        raise NotImplementedError("b200trk optimiser modules: sample_weight must be a tensor or None")
    return f, b, sw


def _iterates(its, losses, compute_losses):
    return [w.unsqueeze(0) for w in its], ([l for l in losses] if compute_losses else [])


class _OptimiserMirror:
    """What the optimiser mirrors share: the seam's claim, and one mirror object per reference module, built again whenever one
    of the module's parameters or scalar settings changes."""

    @classmethod
    def serve(cls, m, weights, feat, bb, sample_weight=None, num_iter=None, compute_losses=True):
        if not (not m.training and _inference(weights, feat, bb) and weights.shape[-1] == 4 and weights.shape[-2] == 4 and
                weights.shape[0] == 1 and (sample_weight is None or isinstance(sample_weight, torch.Tensor))):
            raise NotImplementedError("b200trk %s: eval mode, CUDA float32 tensors, one 4x4 filter" % cls.__name__)
        key = tuple(p._version for p in m.parameters()) + \
            tuple(v for v in vars(m).values() if isinstance(v, (bool, int, float, str, type(None))))
        hit = _state.mirrors.get(m)
        if hit is None or hit[0] != key:
            hit = (key, cls.from_module(m))
            _state.mirrors[m] = hit
        return hit[1].forward(weights, feat, bb, sample_weight, num_iter, compute_losses)

    def __call__(self, *args, **kwargs):
        return self.forward(*args, **kwargs)


class DiMPSteepestDescentGN(_OptimiserMirror):
    """optimizer.py:11-170. Built from the reference module (or its state_dict entries)."""

    def __init__(self, label_map_weight, target_mask_weight, spatial_weight_weight, log_step_length, filter_reg, num_iter=1,
                 feat_stride=16, min_filter_reg=1e-3, alpha_eps=0.0, bin_displacement=0.1):
        self.luts = [t.detach().float().reshape(-1).contiguous() for t in (label_map_weight, target_mask_weight, spatial_weight_weight)]
        self.step_length = float(torch.exp(log_step_length.detach().float()).item())
        self.reg_weight = max(float(filter_reg.detach().float().item()) ** 2, min_filter_reg ** 2)
        self.num_iter, self.feat_stride, self.alpha_eps, self.bin_displacement = num_iter, feat_stride, alpha_eps, bin_displacement

    @classmethod
    def from_module(cls, m):
        # the kernel implements score_act='relu' (LeakyReluPar, activation.py:32-44) and mask_act='sigmoid' (optimizer.py:59-68)
        if type(m.score_activation).__name__ != "LeakyReluPar" or len(m.target_mask_predictor) != 2 or \
                type(m.target_mask_predictor[1]).__name__ != "Sigmoid":
            raise NotImplementedError("b200trk DiMPSteepestDescentGN: only score_act='relu' with mask_act='sigmoid'")
        if m.detach_length != float("Inf") and m.detach_length <= 0:
            raise NotImplementedError("b200trk DiMPSteepestDescentGN: detach_length")
        return cls(m.label_map_predictor.weight, m.target_mask_predictor[0].weight, m.spatial_weight_predictor.weight,
                   m.log_step_length, m.filter_reg, m.num_iter, m.feat_stride, m.min_filter_reg, m.alpha_eps,
                   m.distance_map.bin_displacement)

    def forward(self, weights, feat, bb, sample_weight=None, num_iter=None, compute_losses=True):
        num_iter = self.num_iter if num_iter is None else num_iter
        f, b, sw = _one_sequence(feat, bb, sample_weight)
        luts = [t.to(f.device) for t in self.luts]
        w, its, losses = ops.dimp_sd_gn(weights, f, b, sw, luts[0], luts[1], luts[2], num_iter, self.step_length, self.reg_weight,
                                        self.alpha_eps, self.bin_displacement, self.feat_stride, return_iterates=True,
                                        compute_losses=compute_losses)
        return (w,) + _iterates(its, losses, compute_losses)


class PrDiMPSteepestDescentNewton(_OptimiserMirror):
    """optimizer.py:294-439."""

    def __init__(self, log_step_length, filter_reg, num_iter=1, feat_stride=16, gauss_sigma=1.0, min_filter_reg=1e-3, alpha_eps=0.0,
                 softmax_reg=None, label_shrink=0.0, label_threshold=0.0, normalize_label=False, uni_weight=0.0):
        self.step_length = float(torch.exp(log_step_length.detach().float()).item())
        self.reg_weight = max(float(filter_reg.detach().float().item()) ** 2, min_filter_reg ** 2)
        self.num_iter, self.feat_stride, self.gauss_sigma, self.alpha_eps = num_iter, feat_stride, gauss_sigma, alpha_eps
        self.softmax_reg, self.label_shrink, self.label_threshold = softmax_reg, label_shrink, label_threshold
        self.normalize_label, self.uni_weight = normalize_label, uni_weight

    @classmethod
    def from_module(cls, m):
        return cls(m.log_step_length, m.filter_reg, m.num_iter, m.feat_stride, m.gauss_sigma, m.min_filter_reg, m.alpha_eps,
                   m.softmax_reg, m.label_shrink, m.label_threshold, getattr(m, "normalize_label", False), m.uni_weight)

    def forward(self, weights, feat, bb, sample_weight=None, num_iter=None, compute_losses=True):
        num_iter = self.num_iter if num_iter is None else num_iter
        f, b, sw = _one_sequence(feat, bb, sample_weight)
        w, its, losses = ops.prdimp_sd_newton(weights, f, b, sw, num_iter, self.gauss_sigma, self.step_length, self.reg_weight,
                                              self.alpha_eps, self.softmax_reg, self.label_threshold, self.normalize_label,
                                              self.label_shrink, self.uni_weight, self.feat_stride, return_iterates=True,
                                              compute_losses=compute_losses)
        return (w,) + _iterates(its, losses, compute_losses)


class DiMPL2SteepestDescentGN(_OptimiserMirror):
    """optimizer.py:172-291."""

    def __init__(self, log_step_length, filter_reg, num_iter=1, feat_stride=16, gauss_sigma=1.0, hinge_threshold=-999,
                 min_filter_reg=1e-3, alpha_eps=0.0):
        self.step_length = float(torch.exp(log_step_length.detach().float()).item())
        self.reg_weight = max(float(filter_reg.detach().float().item()) ** 2, min_filter_reg ** 2)
        self.num_iter, self.feat_stride, self.gauss_sigma = num_iter, feat_stride, gauss_sigma
        self.hinge_threshold, self.alpha_eps = hinge_threshold, alpha_eps

    @classmethod
    def from_module(cls, m):
        if m.detach_length != float("Inf") and m.detach_length <= 0:
            raise NotImplementedError("b200trk DiMPL2SteepestDescentGN: detach_length")
        return cls(m.log_step_length, m.filter_reg, m.num_iter, m.feat_stride, m.gauss_sigma, m.hinge_threshold, m.min_filter_reg,
                   m.alpha_eps)

    def forward(self, weights, feat, bb, sample_weight=None, num_iter=None, compute_losses=True):
        num_iter = self.num_iter if num_iter is None else num_iter
        f, b, sw = _one_sequence(feat, bb, sample_weight)
        w, its, losses = ops.dimp_l2_sd_gn(weights, f, b, sw, num_iter, self.gauss_sigma, self.hinge_threshold, self.step_length,
                                           self.reg_weight, self.alpha_eps, self.feat_stride, return_iterates=True,
                                           compute_losses=compute_losses)
        return (w,) + _iterates(its, losses, compute_losses)


# ---------------------------------------------------------------------------------------------------------------
# ltr/models/meta/steepestdescent.py:32-105: GNSteepestDescent over LinearFilterHinge (SuperDiMPSimple / KeepTrack classifiers,
# ltr/models/target_classifier/residual_modules.py:89-135; call site pytracking/tracker/dimp_simple/dimp_simple.py:685-689)
# ---------------------------------------------------------------------------------------------------------------
def _gn_steepest_descent(self, meta_parameter, num_iter=None, *args, **kwargs):
    rm = self.residual_module
    is_list = isinstance(meta_parameter, list)
    w = meta_parameter[0] if is_list and len(meta_parameter) == 1 else meta_parameter
    feat, label, sw = kwargs.get("feat"), kwargs.get("train_label"), kwargs.get("sample_weight")
    act = {"LeakyReluPar": "relu", "BentIdentPar": "bentpar"}.get(type(getattr(rm, "score_activation", None)).__name__)
    if not (type(rm).__name__ == "LinearFilterHinge" and type(rm).__module__.endswith("target_classifier.residual_modules") and
            not args and not self.training and act is not None and isinstance(w, torch.Tensor) and
            set(kwargs) <= {"feat", "bb", "train_label", "sample_weight", "is_distractor"} and kwargs.get("is_distractor") is None and
            _inference(w, feat, label) and w.dim() == 4 and tuple(w.shape[-2:]) == (4, 4) and w.shape[0] == 1 and
            (sw is None or (isinstance(sw, torch.Tensor) and sw.is_cuda)) and self._parameter_batch_dim == 0):
        raise NotImplementedError("b200trk GNSteepestDescent: LinearFilterHinge in eval mode, one 4x4 filter, CUDA float32 tensors")
    f, _, swv = _one_sequence(feat, None, sw)
    n, _, h, wd = f.shape
    if label.numel() != n * (h + 1) * (wd + 1):
        raise NotImplementedError("b200trk GNSteepestDescent: train_label does not match the score map")
    it = self.num_iter if num_iter is None else num_iter
    reg = float(rm.filter_reg.detach().float().item()) if isinstance(rm.filter_reg, torch.Tensor) else float(rm.filter_reg)
    apar = float(rm.score_activation.b) if act == "bentpar" else 1.0      # activation.py:47-55
    wout, its, losses = ops.gn_sd_hinge(w, f, label.reshape(n, 1, h + 1, wd + 1).float(), swv, it, reg, float(rm.hinge_threshold),
                                        float(rm.activation_leak), act, apar, float(self.steplength_reg), return_iterates=True,
                                        compute_losses=bool(self.compute_losses))
    tlist = type(meta_parameter) if is_list else None
    wrap = (lambda t: tlist([t])) if is_list else (lambda t: t)
    iterates = [wrap(its[i:i + 1]) for i in range(it + 1)]
    return wrap(wout), iterates, ([l for l in losses] if self.compute_losses else [])


# ---------------------------------------------------------------------------------------------------------------
# pytracking/libs/optimization.py on the ATOM problems (run(...) updates the variable in place) and ECO's first-frame problem
# ---------------------------------------------------------------------------------------------------------------
def _probe_activation(act):
    """ATOM hands its response activation to the problems as a closure (atom.py:455-468); identify it by evaluation."""
    pts = [-2.0, -0.5, -0.01, 0.0, 0.3, 2.0]
    with torch.no_grad():
        y = act(torch.tensor(pts, dtype=torch.float32).clone())
        floor = -float(act(torch.tensor([-1e4], dtype=torch.float32))[0])
    x = torch.tensor(pts)
    cands = [("none", 0.0, x), ("relu", 0.0, x.clamp(min=0)), ("elu", 1.0, torch.where(x > 0, x, torch.exp(x) - 1))]
    if floor > 0:
        cands.append(("mlu", floor, torch.where(x > 0, x, floor * (torch.exp(x / floor) - 1))))
    for name, par, ref in cands:
        if torch.allclose(y, ref, rtol=1e-5, atol=1e-6):
            return name, par
    return None


class ConjugateGradient:
    """optimization.py:199-289 specialised to ConvProblem (atom/optim.py:71-99): `run(num_cg_iter)` updates `filter` in place."""

    def __init__(self, training_samples, y, filter_reg, sample_weights, filter, response_activation=("mlu", 0.05),
                 fletcher_reeves=True, direction_forget_factor=0):
        if direction_forget_factor != 0:
            raise NotImplementedError("b200trk ConjugateGradient: direction_forget_factor must be 0 (the ATOM default)")
        _check_corr_shape(training_samples, "ConjugateGradient")
        self.x, self.y, self.reg, self.sw, self.filter = training_samples, y, float(filter_reg), sample_weights, filter
        self.act, self.act_param = response_activation if isinstance(response_activation, tuple) else (response_activation, 0.0)
        self.fletcher_reeves = fletcher_reeves

    def run(self, num_cg_iter):
        if num_cg_iter == 0:
            return
        ops.atom_cg_filter(self.filter, self.x, self.y, self.sw, self.reg, num_cg_iter, self.act, self.act_param, self.fletcher_reeves,
                           out=self.filter)


def _single(tlist):
    return len(tlist) == 1 and isinstance(tlist[0], torch.Tensor) and tlist[0].is_cuda and tlist[0].dtype == torch.float32


def _atom_cg_run(self, num_cg_iter):
    p = self.problem
    if not (type(p).__name__ == "ConvProblem" and type(p).__module__.endswith("atom.optim") and not self.debug and
            self.direction_forget_factor == 0 and self.standard_alpha and self.cg_eps == 0.0 and num_cg_iter > 0 and _single(self.x) and
            _single(p.training_samples) and tuple(self.x[0].shape[-2:]) == (4, 4) and self.x[0].shape[0] == 1):
        raise NotImplementedError("b200trk ConjugateGradient.run: ATOM's ConvProblem with one 4x4 filter")
    act = _probe_activation(p.response_activation)
    if act is None:
        raise NotImplementedError("b200trk ConjugateGradient.run: a response activation the kernel does not implement")
    ConjugateGradient(p.training_samples[0], p.y[0], p.filter_reg[0], p.sample_weights[0], self.x[0], act,
                      self.fletcher_reeves).run(num_cg_iter)


def _cg_schedule(num_cg_iter, num_gn_iter):
    """optimization.py:336-339: the CG iteration count of each GN iteration."""
    return [num_cg_iter] * num_gn_iter if isinstance(num_cg_iter, int) and num_gn_iter is not None else num_cg_iter


def _atom_gn_run(self, num_cg_iter, num_gn_iter=None):
    """GaussNewtonCG.run on ATOM's FactorizedConvProblem (atom/optim.py:6-68): the filter and the projection matrix in place."""
    p = self.problem
    # ATOM's problem class only: ECO's first-frame problem (eco/optim.py:8) has the same name and is served by _eco_gn_run
    if not (type(p).__name__ == "FactorizedConvProblem" and type(p).__module__.endswith("atom.optim") and not self.debug and
            not self.analyze_convergence and self.standard_alpha and
            self.cg_eps == 0.0 and self.direction_forget_factor == 0 and len(self.x) == 2 and _single(self.x[:1]) and
            _single(self.x[1:]) and _single(p.training_samples) and tuple(self.x[0].shape[-2:]) == (4, 4) and self.x[0].shape[0] == 1):
        raise NotImplementedError("b200trk GaussNewtonCG.run: ATOM's FactorizedConvProblem with one 4x4 filter")
    its = _cg_schedule(num_cg_iter, num_gn_iter)
    act = _probe_activation(p.response_activation)
    pact = _probe_activation(p.projection_activation)
    if not (isinstance(its, (list, tuple)) and len(its) > 0 and len(set(its)) == 1 and act is not None and pact is not None and
            pact[0] == "none"):
        raise NotImplementedError("b200trk GaussNewtonCG.run: a constant CG schedule, no projection activation")
    _check_corr_shape(p.training_samples[0][:, :16], "GaussNewtonCG.run")
    ops.atom_gn_joint_(self.x[0], self.x[1], p.training_samples[0], p.y[0], p.sample_weights[0], float(p.filter_reg[0]),
                       float(p.projection_reg[0]), int(its[0]), len(its), act[0], act[1], self.fletcher_reeves)


def _eco_gn_run(self, num_cg_iter, num_gn_iter=None):
    """ECO's first-frame joint problem (pytracking/tracker/eco/optim.py:8-117): one launch per feature block."""
    p = self.problem
    if not (type(p).__name__ == "FactorizedConvProblem" and type(p).__module__.endswith("eco.optim") and not self.debug and
            not self.analyze_convergence and self.fletcher_reeves and self.standard_alpha and self.cg_eps == 0.0 and
            self.direction_forget_factor == 0 and len(self.x) % 2 == 0 and len(self.x) > 0):
        raise NotImplementedError("b200trk GaussNewtonCG.run: ECO's FactorizedConvProblem with the default CG settings")
    its = _cg_schedule(num_cg_iter, num_gn_iter)
    nblk = len(self.x) // 2
    ok = isinstance(its, (list, tuple)) and len(its) > 0 and len(set(its)) == 1 and len(p.training_samples) == nblk and \
        getattr(p, "sample_weights_sqrt", None) is not None
    if ok:
        for b in range(nblk):
            hf, pm, xs, rf = self.x[b], self.x[nblk + b], p.training_samples[b], p.reg_filter[b]
            ok = ok and _inference(hf.detach(), pm.detach(), xs, rf, p.diag_M[b]) and hf.dim() == 5 and hf.shape[0] == 1 and \
                hf.shape[-1] == 2 and hf.is_contiguous() and pm.dim() == 2 and xs.dim() == 5 and \
                tuple(xs.shape) == (hf.shape[2], hf.shape[3], xs.shape[2], pm.shape[0], 2) and pm.shape[1] == hf.shape[1] and \
                rf.dim() == 4 and rf.shape[-2] <= min(8, hf.shape[2]) and rf.shape[-1] <= min(8, hf.shape[3]) and \
                p.sample_weights_sqrt[b].numel() in (1, xs.shape[2]) and p.diag_M[b].numel() == hf.numel() // 2 and \
                xs.shape[2] <= 1024 and pm.shape[0] <= 4096 and hf.shape[1] <= 512 and float(p.diag_M[nblk + b]) > 0 and \
                eco_plan.eco_joint_fits(xs.shape[2], pm.shape[0], hf.shape[1])
    if not ok:
        raise NotImplementedError("b200trk GaussNewtonCG.run: ECO feature blocks the joint kernel does not take")
    for b in range(nblk):
        hf, pm, xs = self.x[b], self.x[nblk + b], p.training_samples[b]
        h, wh, n = hf.shape[2], hf.shape[3], xs.shape[2]
        # eco.py:120 slices the projection matrix out of torch.svd's column-major U: run on a row-major copy, write it back
        pc = pm.detach() if pm.is_contiguous() else pm.detach().contiguous()
        ops.eco_joint_gn_(hf.detach(), pc, xs.contiguous(), p.yf[b][..., 0].reshape(1, 1, h, wh).contiguous(),
                          p.sample_weights_sqrt[b].reshape(-1).expand(n).contiguous(), p.reg_filter[b],
                          p.diag_M[b].reshape(1, hf.shape[1], h, wh).contiguous(), float(p.diag_M[nblk + b]),
                          float(p.params.projection_reg), int(its[0]), len(its))
        if pc.data_ptr() != pm.data_ptr():
            pm.detach().copy_(pc)
    self.x.detach_()
    self.clear_temp()
    return self.losses, self.residuals


def gauss_newton_cg_run(reference, *args, **kwargs):
    """ATOM's problem, else ECO's, else the reference; each served path counts under its own name."""
    eco = functools.partial(_serve, "GaussNewtonCG.run[eco]", _eco_gn_run, reference)
    return _serve("GaussNewtonCG.run", _atom_gn_run, eco, *args, **kwargs)


# ---------------------------------------------------------------------------------------------------------------
# pytracking/features/net_wrappers.py:71-75 (extract_backbone) + ltr/models/tracking/dimpnet.py:80-81 (extract_classification_feat)
# ---------------------------------------------------------------------------------------------------------------
class _FeatDict(dict):
    """What the installed `extract_backbone` returns: the reference's layer dict + the classification feature computed in the
    same network pass (served to `extract_classification_feat`)."""
    b200_clf = None


def _arch_of(net):
    """(arch, has_clf_head) when the network is one the engine's plan covers: a reference ResNet backbone to layer3, optionally
    followed by the DiMP classification head (conv(s) + InstanceL2Norm); None otherwise."""
    fe = getattr(net, "feature_extractor", None)
    kind_net = type(net).__name__
    if type(fe).__name__ != "ResNet" or kind_net not in ("DiMPnet", "ToMPnet"):
        return None
    blocks = [len(getattr(fe, "layer%d" % i)) for i in (1, 2, 3)]
    kind = type(fe.layer1[0]).__name__
    arch = {("Bottleneck", (3, 4, 6)): "resnet50", ("Bottleneck", (3, 4, 23)): "resnet101",
            ("BasicBlock", (2, 2, 2)): "resnet18"}.get((kind, tuple(blocks)))
    if arch is None or not set(net.output_layers) <= {"layer2", "layer3"}:
        return None
    if kind_net == "ToMPnet":                  # tompnet.py:141-144: conv3x3 -> InstanceL2Norm on the head layer
        fx = net.head.feature_extractor
        if list(net.head_layer) != ["layer3"] or fx is None or len(fx) != 2 or type(fx[-1]).__name__ != "InstanceL2Norm" or \
                type(fx[0]).__name__ != "Conv2d" or fx[0].bias is not None:
            return arch, False
        return arch, True
    if list(net.classification_layer) != ["layer3"]:
        return None
    head = net.classifier.feature_extractor
    if head is None or type(head[-1]).__name__ != "InstanceL2Norm" or (arch == "resnet101"):
        return None
    return arch, True


def _extract_backbone(self, im):
    net = self.net
    info = _arch_of(net) if (self.use_gpu and self.image_format == "rgb" and im.dim() == 4 and im.shape[1] == 3) else None
    if info is None or torch.is_grad_enabled() or im.shape[0] > 64 or im.shape[-1] % 32 or im.shape[-2] % 32:
        raise NotImplementedError("b200trk extract_backbone: a network the engine covers, RGB crops of multiples of 32, no autograd")
    arch, has_head = info
    per_net = _state.engines.setdefault(net, {})
    key = (int(im.shape[-2]), int(im.shape[-1]))
    eng = per_net.get(key)
    if eng is None or eng.max_batch < im.shape[0]:
        if eng is not None:
            eng.close()
        dev = next(net.parameters()).device
        with torch.cuda.device(dev):
            tomp = type(net).__name__ == "ToMPnet"
            eng = BackboneEngine(net.state_dict(), arch=arch, filter_size=1 if (tomp or not has_head) else net.classifier.filter_size,
                                 max_batch=max(_state.max_batch, int(im.shape[0])), crop_size=key, precision=_state.precision, device=dev,
                                 head=has_head, head_prefix="head.feature_extractor." if tomp else "classifier.feature_extractor.",
                                 norm_scale=float(net.head.feature_extractor[-1].scale) if (tomp and has_head) else None)
        per_net[key] = eng
    want = ("layer2", "layer3", "classification") if has_head else ("layer2", "layer3")
    with torch.cuda.device(eng.device), _timed("extract_backbone"):
        out = eng.forward(im.to(eng.device, dtype=torch.float32, non_blocking=True), want=want)
    feat = _FeatDict((l, out[l]) for l in net.output_layers)
    feat.b200_clf = out.get("classification")
    if type(net).__name__ == "ToMPnet":          # (layer3 tensor, head feature of the same pass) for Head.extract_head_feat
        net._b200_last_feat = (out["layer3"], out.get("classification"))
    _state.last_pass[net] = (eng, [out[l] for l in getattr(net, "bb_regressor_layer", [])], int(im.shape[0]))
    return feat


def _classification_feat(self, backbone_feat):
    clf = getattr(backbone_feat, "b200_clf", None)
    if clf is None:
        raise NotImplementedError("b200trk extract_classification_feat: not the output of the installed extract_backbone")
    return clf


# ---------------------------------------------------------------------------------------------------------------
# ToMP: ltr/models/transformer/heads.py, filter_predictor.py, transformer.py
# ---------------------------------------------------------------------------------------------------------------
def _head_claims(self, feat):
    return isinstance(feat, torch.Tensor) and feat.is_cuda and not torch.is_grad_enabled() and not self.training


def _head_feat_of_last_pass(self, feat, num_sequences=None):
    """Head.extract_head_feat (:54-62) of the crop just extracted: the head feature of the same network pass."""
    if _head_claims(self, feat):
        for net in list(_state.last_pass.keys()):
            if getattr(net, "head", None) is self:
                hit = getattr(net, "_b200_last_feat", None)
                if hit is not None and hit[0] is feat and hit[1] is not None:
                    out = hit[1]
                    return out if num_sequences is None else out.reshape(-1, num_sequences, *out.shape[-3:])
    raise NotImplementedError("b200trk Head.extract_head_feat: not the crop of the last engine pass")


def _head_feat_cached(self, feat, num_sequences=None):
    """Of the stored training frames (tomp.py:289-290 recomputes them every frame): the reference's feature kept by _head_feat_memo."""
    out = _state.head_cache.get(self, {}).get((feat.data_ptr(), tuple(feat.shape), feat._version)) if _head_claims(self, feat) else None
    if out is None:
        raise NotImplementedError("b200trk Head.extract_head_feat: no feature kept for this tensor")
    return out if num_sequences is None else out.reshape(-1, num_sequences, *out.shape[-3:])


def _head_args(self, feat, num_sequences=None):
    return self, feat, num_sequences


def _head_feat_memo(reference, *args, **kwargs):
    """The reference on the caller's arguments; a result the CUDA path would claim is kept until the tensor changes."""
    out = reference(*args, **kwargs)
    self, feat, num_sequences = _head_args(*args, **kwargs)
    if _head_claims(self, feat):
        cache = _state.head_cache.setdefault(self, {})
        if len(cache) > 8:
            cache.clear()
        cache[(feat.data_ptr(), tuple(feat.shape), feat._version)] = out if num_sequences is None else out.reshape(-1, *out.shape[-3:])
    return out


def head_extract_head_feat(reference, *args, **kwargs):
    """The crop just extracted, else a kept feature (each counted by its name), else the reference through _head_feat_memo."""
    memo = functools.partial(_head_feat_memo, reference)
    cached = functools.partial(_serve, "Head.extract_head_feat(cached)", _head_feat_cached, memo)
    return _serve("Head.extract_head_feat", _head_feat_of_last_pass, cached, *args, **kwargs)


def _box_regressor(self, feat, filter):
    """DenseBoxRegressor.forward (:118-141) = filter projection (a 256x256 linear, torch) + 1x1 correlation + the tower on the engine."""
    if not (not self.training and not torch.is_grad_enabled() and isinstance(feat, torch.Tensor) and feat.is_cuda and
            feat.dtype == torch.float32 and feat.dim() == 5 and filter.dim() == 4 and filter.shape[0] == feat.shape[1] and
            filter.shape[-1] == 1 and filter.shape[-2] == 1 and feat.shape[0] * feat.shape[1] <= 4 and
            feat.shape[2] == self.num_channels and len(self.tower) == 12):
        raise NotImplementedError("b200trk DenseBoxRegressor.forward: eval mode, CUDA float32, at most 4 maps, the 12-layer tower")
    from ltr.models.layers import filter as filter_layer
    nf, ns, c, h, w = feat.shape
    filter_proj = self.linear(filter.reshape(-1, c)).reshape(filter.shape) if self.project_filter else filter
    attention = filter_layer.apply_filter(feat, filter_proj)             # (nf, ns, h, w): the 1x1 correlation seam
    key = (h, w)
    per = _state.towers.setdefault(self, {})
    tw = per.get(key)
    if tw is None:
        with torch.cuda.device(feat.device):
            tw = BoxTower(self.state_dict(), h, w, max_batch=4, precision=_state.precision, device=feat.device)
        per[key] = tw
    with _timed("DenseBoxRegressor.forward"):
        ltrb = tw.forward(feat.reshape(nf * ns, c, h, w), attention.reshape(nf * ns, h, w))
    return ltrb.unsqueeze(0)


def _predict_parallel(self, train_feat, test_feat, train_label, num_gth_frames, train_ltrb_target, *args, **kwargs):
    """FilterPredictor.predict_cls_bbreg_filters_parallel (filter_predictor.py:92-150): one kernel assembles the token sequence
    (features + foreground embedding * label + box-encoding MLP); position encoding and key-padding mask are per-shape constants;
    the transformer call goes through the Transformer.forward seam."""
    if train_feat.dim() == 4:
        train_feat = train_feat.unsqueeze(1)
    if test_feat.dim() == 4:
        test_feat = test_feat.unsqueeze(1)
    if train_ltrb_target.dim() == 4:
        train_ltrb_target = train_ltrb_target.unsqueeze(1)
    if not (not self.training and not torch.is_grad_enabled() and all(isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32
                                                                      for t in (train_feat, test_feat, train_ltrb_target)) and
            isinstance(train_label, torch.Tensor) and train_label.is_cuda and train_feat.shape[1] == 1 and test_feat.shape[1] == 1 and
            train_feat.shape[-2:] == test_feat.shape[-2:] and train_feat.shape[2] <= 256 and train_label.dim() == 4 and not args and not kwargs):
        raise NotImplementedError("b200trk predict_cls_bbreg_filters_parallel: eval mode, one sequence of CUDA float32 maps")
    nf_tr, _, c, h, w = train_feat.shape
    nf_te = test_feat.shape[0]
    st = _state.builders.get(self)
    if st is None:
        with torch.cuda.device(train_feat.device):
            st = {"builder": TokenBuilder(self.state_dict(), device=train_feat.device), "const": {}}
        _state.builders[self] = st
    key = (nf_tr, nf_te, h, w, int(num_gth_frames))
    if key not in st["const"]:
        test_pos = self.get_positional_encoding(test_feat).permute(1, 2, 0, 3, 4).flatten(2).permute(2, 0, 1)
        train_pos = self.get_positional_encoding(train_feat).permute(1, 2, 0, 3, 4).flatten(2).permute(2, 0, 1)
        pos = torch.cat([train_pos, test_pos], dim=0).contiguous()
        L = (nf_tr + nf_te) * h * w
        mask = torch.zeros(2, L, dtype=torch.bool)
        mask[1, num_gth_frames * h * w:-h * w] = True
        st["const"] = {key: (pos, mask.to(train_feat.device))}
    pos, mask = st["const"][key]
    feat = st["builder"].build(train_feat[:, 0], test_feat[:, 0], train_label[:, 0].float(), train_ltrb_target[:, 0], B=2,
                               use_test_token=self.use_test_frame_encoding)
    output_embed, enc_mem = self.transformer(feat, mask=mask, query_embed=self.query_embed_fg_decoder.weight, pos_embed=pos)
    stack_shape = (nf_te, 2, c, h, w)
    enc_opt = enc_mem[-h * w:].transpose(0, 1).permute(0, 2, 1).reshape(stack_shape)
    dec_opt = output_embed.squeeze(0).transpose(1, 2).reshape(2, -1, 1, 1)
    return dec_opt[0].unsqueeze(0), dec_opt[1].unsqueeze(0), enc_opt[:, 0].unsqueeze(1), enc_opt[:, 1].unsqueeze(1)


def _transformer(self, src, mask, query_embed, pos_embed):
    """Transformer.forward (transformer.py:90-96): an engine per module and token count."""
    if not (not self.training and _inference(src, query_embed, pos_embed) and src.dim() == 3 and query_embed.shape[0] == 1 and
            self.d_model // self.nhead == 32 and not self.decoder.return_intermediate and
            type(self.encoder.norm).__name__ == "NoneType"):
        raise NotImplementedError("b200trk Transformer.forward: eval mode, CUDA float32, head width 32, no encoder norm")
    key = (int(src.shape[0]), int(src.shape[1]))
    per = _state.tr_engines.setdefault(self, {})
    eng = per.get(key)
    if eng is None:
        with torch.cuda.device(src.device):
            eng = TransformerEngine(self.state_dict(), key[0], key[1], d_model=self.d_model, nhead=self.nhead,
                                    dim_ff=self.encoder.layers[0].linear1.out_features, n_enc=len(self.encoder.layers),
                                    n_dec=len(self.decoder.layers))
        per[key] = eng
    with _timed("Transformer.forward"):
        return eng.forward(src, mask, query_embed, pos_embed)


# ---------------------------------------------------------------------------------------------------------------
# ltr/models/bbreg/atom_iou_net.py
# ---------------------------------------------------------------------------------------------------------------
def _iou_feat(self, feat2):
    """AtomIoUNet.get_iou_feat (:172-179 <- DiMP.get_iou_features dimp.py:318-320): when its input is exactly what the last engine
    pass returned, the four convolutions run on the activations still in the engine's arena."""
    if not torch.is_grad_enabled() and isinstance(feat2, (list, tuple)) and len(feat2) == 2:
        for net, (eng, feats, batch) in list(_state.last_pass.items()):
            if getattr(net, "bb_regressor", None) is self and len(feats) == 2 and feats[0] is feat2[0] and feats[1] is feat2[1] and \
                    list(net.bb_regressor_layer) == ["layer2", "layer3"]:
                if not getattr(eng, "iou_dims", None):
                    eng.attach_iou_head(net.state_dict())
                with torch.cuda.device(eng.device):
                    return eng.iou_features(batch)
    raise NotImplementedError("b200trk AtomIoUNet.get_iou_feat: not the layers of the last engine pass")


class _PredictIoU(torch.autograd.Function):
    """AtomIoUNet.predict_iou (:96-136 <- DiMP.optimize_boxes_* dimp.py:737-742): the tracker differentiates the predicted IoUs
    w.r.t. the proposals with autograd; one library call returns the IoUs and their box gradient, wrapped here so that the tracker's
    own `outputs.backward(...)` / `bb_init.grad` code runs unchanged."""

    @staticmethod
    def forward(ctx, proposals, pred, modulation, feat):
        iou, grad = pred.predict_iou(modulation, feat, proposals.detach(), return_grad=True)
        ctx.save_for_backward(grad.reshape(proposals.shape))
        return iou.reshape(proposals.shape[0], proposals.shape[1])

    @staticmethod
    def backward(ctx, grad_output):
        (g,) = ctx.saved_tensors
        return g * grad_output.unsqueeze(-1), None, None, None


def _predict_iou(self, modulation, feat, proposals):
    if not (not self.training and isinstance(proposals, torch.Tensor) and proposals.is_cuda and proposals.dtype == torch.float32 and
            proposals.dim() == 3 and proposals.shape[0] == 1 and 1 <= proposals.shape[1] <= 16 and len(modulation) == 2 and len(feat) == 2 and
            all(isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and not t.requires_grad
                for t in list(modulation) + list(feat)) and feat[0].shape[0] == 1 and modulation[0].numel() == feat[0].shape[1] and
            type(self.fc3_rt).__name__ == "LinearBlock" and self.fc3_rt.bn is not None and self.fc3_rt.relu is not None):
        raise NotImplementedError("b200trk AtomIoUNet.predict_iou: eval mode, one image, 1-16 CUDA float32 proposals")
    pred = _state.predictors.get(self)
    if pred is None:
        with torch.cuda.device(proposals.device):
            pred = IoUPredictor(self.state_dict(), prefix="", device=proposals.device)
        _state.predictors[self] = pred
    if proposals.requires_grad and torch.is_grad_enabled():
        return _PredictIoU.apply(proposals, pred, modulation, feat)
    return pred.predict_iou(modulation, feat, proposals)


# ---------------------------------------------------------------------------------------------------------------
# `_prroi_pooling`: the three-function native module of ltr/external/PreciseRoIPooling/pytorch/prroi_pool/src/prroi_pooling_gpu.c,
# loaded by functional.py:18-38
# ---------------------------------------------------------------------------------------------------------------
class PrRoIPoolingModule:
    """Drop-in for the pybind module `functional._import_prroi_pooling()` returns (functional.py:21-38).  `previous` is whatever was
    bound at the seam before (None in a stock checkout, whose own module is CUDA-only as well): it keeps serving non-CUDA tensors."""

    def __init__(self, previous=None):
        self.previous = previous

    def _run(self, name, op, features, *args):
        """`op` for CUDA features (prroi_pooling_gpu.c's arguments, ending in pooled_height, pooled_width, spatial_scale)."""
        if not features.is_cuda:
            if self.previous is None:
                raise NotImplementedError("Precise RoI Pooling only supports GPU (cuda) implememtations.")      # functional.py:62-63
            return getattr(self.previous, name + "_cuda")(features, *args)
        *tensors, pooled_height, pooled_width, spatial_scale = args
        _count(name)
        return op(features, *tensors, int(pooled_height), int(pooled_width), float(spatial_scale))

    def prroi_pooling_forward_cuda(self, *args):
        return self._run("prroi_pooling_forward", ops.prroi_pool_forward, *args)

    def prroi_pooling_backward_cuda(self, *args):
        return self._run("prroi_pooling_backward", ops.prroi_pool_backward, *args)

    def prroi_pooling_coor_backward_cuda(self, *args):
        return self._run("prroi_pooling_coor_backward", ops.prroi_pool_coor_backward, *args)


_PRROI = "ltr.external.PreciseRoIPooling.pytorch.prroi_pool.functional"


def import_prroi_pooling(reference):
    """functional.py:21-38: hand out the stand-in bound at `_prroi_pooling` instead of building the reference's own extension."""
    bound = importlib.import_module(_PRROI)._prroi_pooling
    return bound if isinstance(bound, PrRoIPoolingModule) else PrRoIPoolingModule(bound)


# ---------------------------------------------------------------------------------------------------------------
# ECO: pytracking/tracker/eco/optim.py:140-163 (FilterOptim.run, one launch per feature block); eco.py:244-252, 297-300 (the
# score computation: apply_filter, sample_fs as localize_target calls it, preprocess_sample)
# ---------------------------------------------------------------------------------------------------------------
def _eco_block_ok(hf, xs, yf, sw, rf):
    return (_inference(hf, xs, yf, sw, rf) and hf.dim() == 5 and hf.shape[0] == 1 and hf.shape[-1] == 2 and
            hf.shape[1] in (16, 32, 64, 128) and hf.is_contiguous() and xs.is_contiguous() and
            tuple(xs.shape) == (hf.shape[2], hf.shape[3], xs.shape[2], hf.shape[1], 2) and xs.data_ptr() % 16 == 0 and
            yf.numel() == hf.shape[2] * hf.shape[3] and sw.numel() == xs.shape[2] and xs.shape[2] <= 4096 and rf.dim() == 4 and
            rf.shape[-2] <= min(8, hf.shape[2]) and rf.shape[-1] <= min(8, hf.shape[3]))


def _eco_filter_cg(self, num_iter, new_xf=None):
    if num_iter == 0:
        raise NotImplementedError("b200trk FilterOptim.run: no iterations (the reference returns at once)")
    nb = len(self.filter)
    dff = float(self.direction_forget_factor)
    have = self.p is not None and dff != 0
    if not (not self.debug and len(self.training_samples) == nb and len(self.reg_filter) == nb and
            (self.sample_energy is not None or new_xf is not None) and
            all(_eco_block_ok(*b) for b in zip(self.filter, self.training_samples, self.yf, self.sample_weights, self.reg_filter)) and
            (new_xf is None or (len(new_xf) == nb and all(_inference(x) and x.numel() == f.numel() for x, f in zip(new_xf, self.filter)))) and
            (not have or (isinstance(self.rho, list) and len(self.rho) == nb and len(self.p) == nb and
                          (self.fletcher_reeves or self.r_prev is not None)))):
        raise NotImplementedError("b200trk FilterOptim.run: feature blocks the CG kernel does not take")
    tlist = type(self.filter)
    lr = self.params.precond_learning_rate
    if self.sample_energy is not None and not getattr(self, "_b200trk_energy_owned", False):
        # eco.py:168 hands over joint_problem.sample_energy itself; the library updates the energy in place, so take a copy once
        self.sample_energy = tlist([e.detach().clone().contiguous() for e in self.sample_energy])
    energies, ps, rps, rhos = [], [], [], []
    for i in range(nb):
        st = None
        if have:
            st = {"p": self.p[i].contiguous(), "r_prev": None if self.fletcher_reeves else self.r_prev[i].contiguous(),
                  "rho": self.rho[i].detach().to(self.filter[i].device, torch.float32).reshape(1).clone()}
        e, st = ops.eco_filter_cg_(self.filter[i], self.training_samples[i], self.yf[i], self.sample_weights[i], self.reg_filter[i],
                                   None if self.sample_energy is None else self.sample_energy[i], num_iter,
                                   None if new_xf is None else new_xf[i], st, self.fletcher_reeves, self.standard_alpha, dff,
                                   float(lr[i]) if isinstance(lr, (list, tuple)) else float(lr),
                                   float(self.params.precond_data_param), float(self.params.precond_reg_param))
        energies.append(e)
        ps.append(st["p"])
        rps.append(st["r_prev"])
        rhos.append(st["rho"].reshape(()))
    # the state stays in the reference's own attributes and layout, so a later fall-through run continues from it
    self.sample_energy = tlist(energies)
    self._b200trk_energy_owned = True
    self.p, self.rho = tlist(ps), tlist(rhos)
    self.r_prev = None if self.fletcher_reeves else tlist(rps)


def _eco_apply_filter(self, sample_xf):
    filt = self.filter
    if not (len(filt) == len(sample_xf) and all(_inference(f, x) and f.dim() == 5 and x.dim() == 5 and f.shape[0] == 1 and f.shape[-1] == 2 and
                                                tuple(x.shape[1:]) == tuple(f.shape[1:]) for f, x in zip(filt, sample_xf))):
        raise NotImplementedError("b200trk ECO.apply_filter: one CUDA float32 filter per sample block")
    return type(sample_xf)([ops.eco_apply_filter(f.contiguous(), x.contiguous()) for f, x in zip(filt, sample_xf)])


def _eco_preprocess_sample(self, x):
    win, ifs = self.window, self.interp_fs

    def ok(e, w, bf):
        if not (_inference(e, w) and e.dim() == 4 and min(e.stride()) >= 0 and isinstance(bf, (tuple, list)) and len(bf) == 2 and
                _inference(bf[0], bf[1])):
            return False
        h, wd = e.shape[2], e.shape[3]
        return (w.numel() == h * wd and bf[0].numel() == 2 * (h + (h + 1) % 2) and bf[1].numel() == 2 * (wd // 2 + 1) and
                4 * (h * wd + 1 + 2 * (h * (wd // 2 + 1) + h + wd)) <= 200 * 1024)
    if not (len(x) == len(win) == len(ifs) and all(ok(e, w, bf) for e, w, bf in zip(x, win, ifs))):
        raise NotImplementedError("b200trk ECO.preprocess_sample: feature blocks the kernel does not take")
    return type(x)([ops.eco_preprocess_sample_(e, w.contiguous(), bf[0].contiguous(), bf[1].contiguous())
                    for e, w, bf in zip(x, win, ifs)])


def _eco_sample_fs(a, grid_sz=None, rescale=True):
    if isinstance(a, torch.Tensor) and grid_sz is not None and rescale and _inference(a) and a.dim() == 5 and a.shape[1] == 1 and \
            a.shape[-1] == 2 and a.shape[2] % 2 == 1:
        oh, ow = int(grid_sz[0]), int(grid_sz[1])
        if float(grid_sz[0]) == oh and float(grid_sz[1]) == ow and oh >= a.shape[2] and ow >= 2 * a.shape[3] - 1 and \
                (oh, ow) != (a.shape[2], 2 * a.shape[3] - 1):
            return ops.eco_sample_fs(a.contiguous(), (oh, ow))
    raise NotImplementedError("b200trk fourier.sample_fs: one summed CUDA float32 series on a larger integer grid")


def _eco_shift_fs(a, shift):
    if not (isinstance(a, torch.Tensor) and _inference(a) and a.dim() == 5 and a.shape[-1] == 2 and a.shape[2] % 2 == 1 and a.numel() > 0):
        raise NotImplementedError("b200trk fourier.shift_fs: a CUDA float32 Fourier series")
    sy, sx = float(shift[0]), float(shift[1])
    if sy == 0 and sx == 0:
        raise NotImplementedError("b200trk fourier.shift_fs: a zero shift returns its argument (fourier.py:86-87)")
    return ops.eco_shift_fs(a.contiguous(), sy, sx)


class _EcoFourier:
    """`fourier` as the ECO module sees it: sample_fs of one summed series on a larger grid (eco.py:249-252) and shift_fs
    (eco.py:119-127, 226-227) go to the library, every other name and every call they do not claim is the reference module's
    (other trackers keep theirs untouched)."""

    def __init__(self, reference):
        self.reference = reference

    def __getattr__(self, name):
        return getattr(self.reference, name)

    def sample_fs(self, *args, **kwargs):
        return _serve("fourier.sample_fs[eco]", _eco_sample_fs, self.reference.sample_fs, *args, **kwargs)

    def shift_fs(self, a, shift):
        if isinstance(a, (list, tuple)) and not isinstance(a, torch.Tensor):                 # @tensor_operation: element-wise over a TensorList
            return type(a)([self.shift_fs(e, shift) for e in a])
        return _serve("fourier.shift_fs[eco]", _eco_shift_fs, self.reference.shift_fs, a, shift)


# ---------------------------------------------------------------------------------------------------------------
# install(): rebind every seam of SURVEY.md 8(b) inside an importable, unmodified pytracking / ltr checkout
# ---------------------------------------------------------------------------------------------------------------
# (reference module, owner class or None for the module itself, attribute, seam, optional, tensor_operation): a seam function is bound
# through a wrapper handing it the reference, made element-wise over TensorLists by @tensor_operation where the reference function is;
# a class is instantiated with the reference; an optional module that does not import is left out.
SEAMS = [
    ("ltr.models.layers.filter", None, "apply_filter", _seam("apply_filter", _served_apply_filter), False, False),
    ("ltr.models.layers.filter", None, "apply_feat_transpose",
     _seam("apply_feat_transpose", _served_apply_feat_transpose), False, False),
    ("pytracking.libs.dcf", None, "max2d", _seam("max2d", _served_max2d), False, False),
    ("ltr.models.target_classifier.optimizer", "DiMPSteepestDescentGN", "forward",
     _seam("DiMPSteepestDescentGN.forward", DiMPSteepestDescentGN.serve), False, False),
    ("ltr.models.target_classifier.optimizer", "PrDiMPSteepestDescentNewton", "forward",
     _seam("PrDiMPSteepestDescentNewton.forward", PrDiMPSteepestDescentNewton.serve), False, False),
    ("ltr.models.target_classifier.optimizer", "DiMPL2SteepestDescentGN", "forward",
     _seam("DiMPL2SteepestDescentGN.forward", DiMPL2SteepestDescentGN.serve), False, False),
    ("ltr.models.meta.steepestdescent", "GNSteepestDescent", "forward",
     _seam("GNSteepestDescent.forward", _gn_steepest_descent), True, False),
    ("pytracking.features.net_wrappers", "NetWithBackbone", "extract_backbone",
     _seam("extract_backbone", _extract_backbone), False, False),
    ("ltr.models.tracking.dimpnet", "DiMPnet", "extract_classification_feat",
     _seam("extract_classification_feat", _classification_feat), False, False),
    ("ltr.models.transformer.heads", "Head", "extract_head_feat", head_extract_head_feat, False, False),
    ("ltr.models.transformer.heads", "DenseBoxRegressor", "forward", _seam("DenseBoxRegressor.forward", _box_regressor), False, False),
    ("ltr.models.transformer.filter_predictor", "FilterPredictor", "predict_cls_bbreg_filters_parallel",
     _seam("FilterPredictor.predict_cls_bbreg_filters_parallel", _predict_parallel), False, False),
    ("ltr.models.bbreg.atom_iou_net", "AtomIoUNet", "get_iou_feat", _seam("get_iou_feat", _iou_feat), False, False),
    ("ltr.models.bbreg.atom_iou_net", "AtomIoUNet", "predict_iou", _seam("predict_iou", _predict_iou), False, False),
    (_PRROI, None, "_prroi_pooling", PrRoIPoolingModule, False, False),
    (_PRROI, None, "_import_prroi_pooling", import_prroi_pooling, False, False),
    ("pytracking.libs.operation", None, "conv2d", operation_conv2d, False, True),
    ("pytracking.libs.operation", None, "conv1x1", _seam("operation.conv1x1", conv1x1), False, True),
    ("pytracking.libs.optimization", "ConjugateGradient", "run", _seam("ConjugateGradient.run", _atom_cg_run), False, False),
    ("pytracking.libs.optimization", "GaussNewtonCG", "run", gauss_newton_cg_run, False, False),
    ("pytracking.tracker.eco.optim", "FilterOptim", "run", _seam("FilterOptim.run", _eco_filter_cg), True, False),
    ("pytracking.tracker.eco.eco", "ECO", "apply_filter", _seam("ECO.apply_filter", _eco_apply_filter), True, False),
    ("pytracking.tracker.eco.eco", "ECO", "preprocess_sample", _seam("ECO.preprocess_sample", _eco_preprocess_sample), True, False),
    ("pytracking.tracker.eco.eco", None, "fourier", _EcoFourier, True, False),
    ("ltr.models.transformer.transformer", "Transformer", "forward", _seam("Transformer.forward", _transformer), False, False),
]

_installed = []          # [(owner object, attribute name, original value)]


def _bind(seam, reference, tensor_operation):
    def bound(*args, **kwargs):
        return seam(reference, *args, **kwargs)
    if tensor_operation:
        bound = importlib.import_module("pytracking.libs.tensorlist").tensor_operation(bound)
    return bound


def install(max_batch=16, precision=0, skip=()):
    """`skip`: attribute names (e.g. "predict_iou" or "AtomIoUNet.predict_iou") to leave on the reference implementation.
    Rebind the seams inside an importable pytracking / ltr checkout (no reference file is edited); `uninstall()` restores them.
    Calls the CUDA path does not claim (CPU tensors, autograd, training mode, shapes the library rejects) fall through to the
    reference implementation. Returns the list of rebound attributes."""
    global _state
    if not _installed:
        _state = _State(max_batch, precision)
        for module, owner, name, seam, optional, tensor_operation in SEAMS:
            try:
                mod = importlib.import_module(module)
            except Exception:
                if optional:
                    continue
                raise
            obj = getattr(mod, owner) if owner else mod
            if name in skip or "%s.%s" % (obj.__name__, name) in skip:
                continue
            reference = obj.__dict__[name] if isinstance(obj, type) else getattr(obj, name)
            _installed.append((obj, name, reference))
            setattr(obj, name, seam(reference) if isinstance(seam, type) else _bind(seam, reference, tensor_operation))
    return ["%s.%s" % (o.__name__, n) for o, n, _ in _installed]


def uninstall():
    """Restore every attribute `install()` rebound and release the engines and caches it built."""
    global _state
    while _installed:
        owner, name, orig = _installed.pop()
        setattr(owner, name, orig)
    _state = None
