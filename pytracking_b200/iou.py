"""IoUNet box refinement through the C ABI (`b200trk_iou_*`, csrc/iou_refine.cu): `IoUPredictor` mirrors
`AtomIoUNet.predict_iou` (ltr/models/bbreg/atom_iou_net.py:96-136) and the box optimisation loops of
`DiMP.optimize_boxes_default / _relative` (pytracking/tracker/dimp/dimp.py:725-793), with the box gradient written out instead of
obtained by autograd.  Built once from the bb_regressor's state_dict entries."""
import ctypes as C

import torch

from . import _lib


class IoUModulation:
    """AtomIoUNet.get_modulation (atom_iou_net.py:138-170) after conv3_1r / conv4_1r (BackboneEngine.attach_iou_ref): the fc3_1r,
    fc34_3r and fc34_4r blocks of the bb_regressor's state_dict, BN folded at create time."""

    def __init__(self, state_dict, prefix="bb_regressor.", device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("IoUModulation: CUDA device required (the engine has no CPU path)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        keep = []

        def hp(key):
            t = state_dict[prefix + key].detach().float().contiguous().cpu()
            keep.append(t)
            return t

        def block(name):
            w = hp(name + ".0.weight")
            b = _lib.LinearBlock(w.data_ptr(), hp(name + ".0.bias").data_ptr(), hp(name + ".1.weight").data_ptr(),
                                 hp(name + ".1.bias").data_ptr(), hp(name + ".1.running_mean").data_ptr(),
                                 hp(name + ".1.running_var").data_ptr())
            return b, w.shape
        b31, s31 = block("fc3_1r")
        b3, s3 = block("fc34_3r")
        b4, s4 = block("fc34_4r")
        self.C3 = int(state_dict[prefix + "conv3_1r.0.weight"].shape[0])
        self.C4 = int(state_dict[prefix + "conv4_1r.0.weight"].shape[0])
        self.D, self.M3, self.M4 = int(s31[0]), int(s3[0]), int(s4[0])
        if tuple(s31[1:]) != (self.C3, 3, 3) or s3[1] != self.D + self.C4 or s4[1] != self.D + self.C4:
            raise RuntimeError("IoUModulation: unexpected bb_regressor shapes %s %s %s" % (tuple(s31), tuple(s3), tuple(s4)))
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_iou_modulation_create(C.byref(h), C.byref(b31), C.byref(b3), C.byref(b4), self.C3, self.C4,
                                                                self.D, self.M3, self.M4), "iou_modulation_create")
        self.handle = h
        del keep

    def get(self, backbone, s, boxes, images=None):
        """get_modulation of boxes [R,4] (x, y, w, h; box r on image images[r], default r) on the layer2 / layer3 activations of the last
        forward pass (batch s) of `backbone` -> (mod3 [R,M3], mod4 [R,M4]) CUDA tensors."""
        b = torch.as_tensor(boxes, dtype=torch.float32).reshape(-1, 4).contiguous().cpu()
        R = b.shape[0]
        img = None if images is None else (C.c_int * R)(*[int(i) for i in images])
        m3 = torch.empty(R, self.M3, device=self.device, dtype=torch.float32)
        m4 = torch.empty(R, self.M4, device=self.device, dtype=torch.float32)
        _lib.check(_lib.lib().b200trk_iou_modulation_get(self.handle, backbone.handle, int(s), R, img, C.c_void_p(b.data_ptr()),
                                                         C.c_void_p(m3.data_ptr()), C.c_void_p(m4.data_ptr()),
                                                         C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)),
                   "iou_modulation_get")
        return m3, m4

    def close(self):
        if getattr(self, "handle", None):
            _lib.lib().b200trk_iou_modulation_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class IoUPredictor:
    def __init__(self, state_dict, prefix="bb_regressor.", device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("IoUPredictor: CUDA device required (the engine has no CPU path)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        keep = []

        def hp(key):
            t = state_dict[prefix + key].detach().float().contiguous().cpu()
            keep.append(t)
            return t

        def block(name):
            w = hp(name + ".linear.weight")
            b = _lib.LinearBlock(w.data_ptr(), hp(name + ".linear.bias").data_ptr(), hp(name + ".bn.weight").data_ptr(),
                                 hp(name + ".bn.bias").data_ptr(), hp(name + ".bn.running_mean").data_ptr(),
                                 hp(name + ".bn.running_var").data_ptr())
            return b, w.shape
        b3, s3 = block("fc3_rt")
        b4, s4 = block("fc4_rt")
        wp, bp = hp("iou_predictor.weight"), hp("iou_predictor.bias")
        self.C3 = state_dict[prefix + "conv3_2t.0.weight"].shape[0]
        self.C4 = state_dict[prefix + "conv4_2t.0.weight"].shape[0]
        self.P3 = int(round((s3[1] // self.C3) ** 0.5))
        self.P4 = int(round((s4[1] // self.C4) ** 0.5))
        self.D3, self.D4 = int(s3[0]), int(s4[0])
        assert self.C3 * self.P3 ** 2 == s3[1] and self.C4 * self.P4 ** 2 == s4[1] and wp.numel() == self.D3 + self.D4
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_iou_predictor_create(C.byref(h), C.byref(b3), C.byref(b4), C.c_void_p(wp.data_ptr()),
                                                               C.c_void_p(bp.data_ptr()), self.C3, self.P3, self.C4, self.P4, self.D3,
                                                               self.D4), "iou_predictor_create")
        self.handle = h
        del keep

    @staticmethod
    def _dev(t, name):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
            raise RuntimeError("IoUPredictor: '%s' must be a CUDA float32 tensor" % name)
        return t.contiguous()

    def _args(self, modulation, feat):
        m3, m4 = self._dev(modulation[0].reshape(-1), "modulation[0]"), self._dev(modulation[1].reshape(-1), "modulation[1]")
        f3, f4 = self._dev(feat[0], "feat[0]"), self._dev(feat[1], "feat[1]")
        f3, f4 = f3.reshape(-1, *f3.shape[-2:]), f4.reshape(-1, *f4.shape[-2:])
        if m3.numel() != self.C3 or m4.numel() != self.C4 or f3.shape[0] != self.C3 or f4.shape[0] != self.C4:
            raise RuntimeError("IoUPredictor: one image per call (modulation [C], features [1,C,H,W])")
        return m3, m4, f3, f4

    def predict_iou(self, modulation, feat, proposals, return_grad=False):
        """proposals [1,R,4] or [R,4] (x,y,w,h) -> iou [1,R] (and d iou / d proposals [1,R,4])."""
        m3, m4, f3, f4 = self._args(modulation, feat)
        p = self._dev(proposals.reshape(-1, 4), "proposals")
        r = p.shape[0]
        iou = torch.empty(r, device=p.device)
        grad = torch.empty(r, 4, device=p.device) if return_grad else None
        _lib.check(_lib.lib().b200trk_iou_predict(
            self.handle, C.c_void_p(m3.data_ptr()), C.c_void_p(m4.data_ptr()), C.c_void_p(f3.data_ptr()), f3.shape[1], f3.shape[2],
            C.c_void_p(f4.data_ptr()), f4.shape[1], f4.shape[2], C.c_void_p(p.data_ptr()), r, C.c_void_p(iou.data_ptr()),
            C.c_void_p(grad.data_ptr()) if grad is not None else None, C.c_void_p(torch.cuda.current_stream().cuda_stream)), "iou_predict")
        return (iou.reshape(1, r), grad.reshape(1, r, 4)) if return_grad else iou.reshape(1, r)

    def refine(self, modulation, feat, init_boxes, num_iter, step_length, step_decay=1.0, relative=False):
        """DiMP.optimize_boxes_default / _relative: init_boxes [R,4] -> (boxes [R,4], iou [R]) as CUDA tensors."""
        m3, m4, f3, f4 = self._args(modulation, feat)
        b = self._dev(init_boxes.reshape(-1, 4), "init_boxes").clone()
        r = b.shape[0]
        iou = torch.empty(r, device=b.device)
        _lib.check(_lib.lib().b200trk_iou_refine(
            self.handle, C.c_void_p(m3.data_ptr()), C.c_void_p(m4.data_ptr()), C.c_void_p(f3.data_ptr()), f3.shape[1], f3.shape[2],
            C.c_void_p(f4.data_ptr()), f4.shape[1], f4.shape[2], C.c_void_p(b.data_ptr()), r, int(num_iter), float(step_length),
            float(step_decay), int(bool(relative)), C.c_void_p(iou.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
            "iou_refine")
        return b, iou

    def close(self):
        if getattr(self, "handle", None):
            _lib.lib().b200trk_iou_predictor_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
