"""Per-sequence DiMP frame engine over the C ABI's host-buffer calls (`b200trk_dimp_*`, include/b200trk.h).

One object = one tracked sequence on one GPU: network handle + online-model state (sample memory, boxes,
weights, filter) living in HBM for the whole sequence.  The host side only does what the reference tracker
does on the host (pytracking/tracker/dimp/dimp.py): localisation decisions on the 19x19 score map and the
sample-weight bookkeeping; every tensor op runs in the CUDA library.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .engine import BackboneEngine


class _DevView:
    """Zero-copy torch view of a device buffer owned by the C library."""

    def __init__(self, ptr, shape, owner):
        self._owner = owner
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False), "version": 3,
                                         "strides": None}


def _view(ptr, shape, owner, device, plane_pitch=None):
    """plane_pitch: floats between two [H,W] planes of a [n,C,H,W] buffer (None = dense) -> a strided view, no copy."""
    if plane_pitch is None or plane_pitch == shape[-1] * shape[-2]:
        return torch.as_tensor(_DevView(ptr, shape, owner), device=device)
    n, c, h, w = shape
    flat = torch.as_tensor(_DevView(ptr, (n * c * plane_pitch,), owner), device=device)
    return flat.as_strided((n, c, h, w), (c * plane_pitch, plane_pitch, w, 1))


class SampleWeights:
    """Host mirror of DiMP.update_sample_weights (pytracking/tracker/dimp/dimp.py:445-484), float32 arithmetic."""

    def __init__(self, memory_size, num_init, learning_rate=0.01, init_samples_minimum_weight=0.25):
        self.w = np.zeros(memory_size, dtype=np.float32)
        self.w[:num_init] = np.float32(1.0) / np.float32(num_init)
        self.num_init = num_init
        self.num_stored = num_init
        self.prev_ind = None
        self.lr = learning_rate
        self.min_init = init_samples_minimum_weight if init_samples_minimum_weight else None

    def step(self, learning_rate=None):
        """Returns the memory slot to overwrite and updates the weights in place."""
        lr = np.float32(self.lr if learning_rate is None else learning_rate)
        w = self.w
        s_ind = 0 if self.min_init is None else self.num_init
        if self.num_stored == 0 or lr == 1:
            w[:] = 0
            w[0] = 1
            r_ind = 0
        else:
            if self.num_stored < w.shape[0]:
                r_ind = self.num_stored
            else:
                r_ind = int(np.argmin(w[s_ind:])) + s_ind
            if self.prev_ind is None:
                w /= (np.float32(1) - lr)
                w[r_ind] = lr
            else:
                w[r_ind] = w[self.prev_ind] / (np.float32(1) - lr)
        w /= w.sum(dtype=np.float32)
        if self.min_init is not None and w[:self.num_init].sum(dtype=np.float32) < self.min_init:
            w /= np.float32(self.min_init) + w[self.num_init:].sum(dtype=np.float32)
            w[:self.num_init] = np.float32(self.min_init) / np.float32(self.num_init)
        self.prev_ind = r_ind
        if self.num_stored < w.shape[0]:
            self.num_stored += 1
        return r_ind


def newton_scalars(state_dict, nw):
    """(step_length, reg_weight) of PrDiMPSteepestDescentNewton in float32, as its parameters give them: exp(log_step_length) and
    (filter_reg^2).clamp(min=min_filter_reg^2) (optimizer.py:378-379).  log_step_length / filter_reg come from the state_dict when it
    carries them (a trained net), else from the constructor arguments; params.filter_reg (nw['filter_reg_override']) replaces both
    filter_reg and min_filter_reg, as DiMP._overwrite_classifier_params does (dimp.py:598-600)."""
    po = "classifier.filter_optimizer."
    one = torch.ones(1)
    log_step = state_dict[po + "log_step_length"].float().cpu() if po + "log_step_length" in state_dict else \
        math.log(nw["init_step_length"]) * one
    if nw.get("filter_reg_override") is not None:
        freg = nw["filter_reg_override"] * one
    elif po + "filter_reg" in state_dict:
        freg = state_dict[po + "filter_reg"].float().cpu()
    else:
        freg = nw["init_filter_reg"] * one
    return float(torch.exp(log_step).item()), float((freg * freg).clamp(min=nw["min_filter_reg"] ** 2).item())


def optimizer_args(state_dict, newton):
    """The online optimiser's arguments after `filter_size` of b200trk_dimp_state_create / b200trk_dimp_batch_create (newton=None:
    DiMPSteepestDescentGN over the state_dict's three LUTs) or of b200trk_prdimp_state_create / b200trk_prdimp_batch_create (newton:
    PrDiMPSteepestDescentNewton arguments as newton_hparams returns them), followed by the optimiser's step_length and reg_weight.
    The GN optimiser's bin_displacement, feat_stride, min_filter_reg and alpha_eps are DiMP-50's 0.1, 16, 1e-3 and 0."""
    po = "classifier.filter_optimizer."
    if newton is None:
        luts = [state_dict[po + k].detach().float().reshape(-1).cpu().numpy() for k in
                ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
        step_length = float(torch.exp(state_dict[po + "log_step_length"].float()).item())
        reg_weight = max(float(state_dict[po + "filter_reg"].float().item()) ** 2, 1e-3 ** 2)
        args = [(C.c_float * t.size).from_buffer_copy(t) for t in luts] + [luts[0].size, 0.1, 16.0, step_length, reg_weight, 0.0]
    else:
        step_length, reg_weight = newton_scalars(state_dict, newton)
        sreg = newton["softmax_reg"]
        args = [float(newton["gauss_sigma"]), float(newton["feat_stride"]), step_length, reg_weight, float(newton["alpha_eps"]),
                int(sreg is not None), 0.0 if sreg is None else float(sreg), float(newton["label_threshold"]),
                int(bool(newton["normalize_label"])), float(newton["label_shrink"]), float(newton["init_uni_weight"] or 0.0)]
    return args, step_length, reg_weight


class DiMPFrameEngine:
    def __init__(self, state_dict, arch="resnet50", filter_size=4, memory_size=50, max_batch=1, crop_size=288, precision=0, device=None,
                 newton=None):
        """newton: None for DiMP (DiMPSteepestDescentGN over the three LUTs of the state_dict), or a dict of
        PrDiMPSteepestDescentNewton constructor arguments (tracker.NEWTON_DEFAULTS names) for PrDiMP; the GN keys are then not read.
        A state_dict that carries the optimiser's learnt log_step_length / filter_reg (a trained PrDiMP net) supplies those two."""
        self.backbone = BackboneEngine(state_dict, arch, filter_size, max_batch, crop_size, precision, device)
        self.device = self.backbone.device
        self.memory_size, self.filter_size, self.max_batch = memory_size, filter_size, max_batch
        if newton is not None:
            from .tracker import newton_hparams
            newton = newton_hparams(newton)
        self.newton = newton
        args, self.step_length, self.reg_weight = optimizer_args(state_dict, newton)
        create = "dimp_state_create" if newton is None else "prdimp_state_create"
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(getattr(_lib.lib(), "b200trk_" + create)(C.byref(h), self.backbone.handle, memory_size, filter_size, *args), create)
        self.state = h
        L = _lib.lib()
        cc, hc, wc = self.backbone.dims[6:9]
        self.feat_dims = (cc, hc, wc)
        self.out_sz = (hc + (filter_size + 1) % 2, wc + (filter_size + 1) % 2)
        dev = self.device
        self.filter = _view(L.b200trk_dimp_state_filter(h), (1, cc, filter_size, filter_size), self, dev)
        self.memory = _view(L.b200trk_dimp_state_memory(h), (memory_size, cc, hc, wc), self, dev, L.b200trk_dimp_state_memory_pitch(h))
        self.boxes = _view(L.b200trk_dimp_state_boxes(h), (memory_size, 4), self, dev)
        self.sample_weights = _view(L.b200trk_dimp_state_sample_weights(h), (memory_size,), self, dev)
        self.clf = _view(L.b200trk_dimp_state_clf(h), (max_batch, cc, hc, wc), self, dev)
        self.scores = _view(L.b200trk_dimp_state_scores(h), (max_batch,) + self.out_sz, self, dev)
        # pinned host staging for the per-frame results and update inputs
        self.h_scores = torch.empty((max_batch,) + self.out_sz, dtype=torch.float32).pin_memory()
        self.h_maxval = torch.empty(max_batch, dtype=torch.float32).pin_memory()
        self.h_maxidx = torch.empty(max_batch, 2, dtype=torch.int64).pin_memory()
        self.h_box = torch.empty(4, dtype=torch.float32).pin_memory()
        self.h_sw = torch.empty(memory_size, dtype=torch.float32).pin_memory()
        self._np_scores = self.h_scores.numpy()
        self._np_maxval = self.h_maxval.numpy()
        self._np_maxidx = self.h_maxidx.numpy()

    # ---- per-frame calls ---------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def localize(self, crop_host):
        """crop_host: [S,3,H,W] float32 HOST tensor (pinned), pixel range 0..255.
        H2D + backbone + head + classify + arg-max + D2H; returns numpy views (scores [S,Ho,Wo], max [S], idx [S,2])."""
        s = crop_host.shape[0]
        _lib.check(_lib.lib().b200trk_dimp_localize_host(
            self.state, C.c_void_p(crop_host.data_ptr()), s, C.c_void_p(self.h_scores.data_ptr()),
            C.c_void_p(self.h_maxval.data_ptr()), C.c_void_p(self.h_maxidx.data_ptr()), self._stream()), "dimp_localize_host")
        return self._np_scores[:s], self._np_maxval[:s], self._np_maxidx[:s]

    def localize_device(self, crop_dev, read_back=False):
        """Same device work with the crop already resident in HBM (no host copies unless read_back)."""
        L = _lib.lib()
        s = crop_dev.shape[0]
        cc, hc, wc = self.feat_dims
        _lib.check(L.b200trk_net_forward(self.backbone.handle, C.c_void_p(crop_dev.data_ptr()), s, None, None,
                                         C.c_void_p(self.clf.data_ptr()), self._stream()), "net_forward")
        if not hasattr(self, "_d_maxval"):
            self._d_maxval = torch.empty(self.max_batch, device=self.device, dtype=torch.float32)
            self._d_maxidx = torch.empty(self.max_batch, 2, device=self.device, dtype=torch.int64)
        _lib.check(L.b200trk_apply_filter(C.c_void_p(self.clf.data_ptr()), C.c_void_p(self.filter.data_ptr()),
                                          C.c_void_p(self.scores.data_ptr()), s, cc, hc, wc, self.filter_size,
                                          C.c_void_p(self._d_maxval.data_ptr()), C.c_void_p(self._d_maxidx.data_ptr()),
                                          self._stream()), "apply_filter")
        if read_back:
            return self._d_maxval[:s].cpu(), self._d_maxidx[:s].cpu()
        return None

    def update(self, scale_ind, replace_ind, target_box, sample_weights, n_stored, num_iter):
        """Store the last crop's feature in memory slot `replace_ind` and run `num_iter` SD iterations (asynchronous)."""
        self.h_box.numpy()[:] = target_box
        self.h_sw.numpy()[:n_stored] = sample_weights[:n_stored]
        _lib.check(_lib.lib().b200trk_dimp_update_host(
            self.state, int(scale_ind), int(replace_ind), C.c_void_p(self.h_box.data_ptr()), C.c_void_p(self.h_sw.data_ptr()),
            int(n_stored), int(num_iter), self._stream()), "dimp_update_host")

    def close(self):
        if getattr(self, "state", None):
            _lib.lib().b200trk_dimp_state_destroy(self.state)
            self.state = None
        self.backbone.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
