"""Stage-1 engine handle: the backbone + classification head of a DiMP-style network, built once from a
reference-format state_dict (what `NetWrapper.load_network` produces, pytracking/features/net_wrappers.py:30-37)
and run through the C ABI (`b200trk_net_*`)."""
import ctypes as C
import math
from collections import OrderedDict

import torch

from . import _lib
from .synth import RESNET_ARCH

ARCH_ID = {"resnet18": 18, "resnet50": 50, "resnet101": 101}


def _conv_entry(sd, keep, wkey, bnprefix, stride, pad, bias_key=None):
    w = sd[wkey].detach().float().contiguous().cpu()
    d = _lib.ConvDesc()
    keep.append(w)
    d.weight = w.data_ptr()
    d.bias = 0
    if bias_key is not None and bias_key in sd:
        b = sd[bias_key].detach().float().contiguous().cpu()
        keep.append(b)
        d.bias = b.data_ptr()
    if bnprefix is not None:
        for field, suffix in (("bn_gamma", ".weight"), ("bn_beta", ".bias"), ("bn_mean", ".running_mean"), ("bn_var", ".running_var")):
            t = sd[bnprefix + suffix].detach().float().contiguous().cpu()
            keep.append(t)
            setattr(d, field, t.data_ptr())
    d.cout, d.cin, d.k = int(w.shape[0]), int(w.shape[1]), int(w.shape[2])
    d.stride, d.pad = stride, pad
    return d


def conv_descs_from_state_dict(sd, arch, backbone_prefix="feature_extractor.", head_prefix="classifier.feature_extractor.", head=True):
    """Conv descriptors in the execution order `b200trk_net_create` expects (include/b200trk.h)."""
    block, layers = RESNET_ARCH[arch]
    keep, descs = [], []
    p = backbone_prefix
    descs.append(_conv_entry(sd, keep, p + "conv1.weight", p + "bn1", 2, 3))
    for li in range(3):
        for bi in range(layers[li]):
            q = "%slayer%d.%d." % (p, li + 1, bi)
            stride = 2 if (li > 0 and bi == 0) else 1
            has_ds = (q + "downsample.0.weight") in sd
            if block == "bottleneck":
                descs.append(_conv_entry(sd, keep, q + "conv1.weight", q + "bn1", 1, 0))
                descs.append(_conv_entry(sd, keep, q + "conv2.weight", q + "bn2", stride, 1))
                if has_ds:
                    descs.append(_conv_entry(sd, keep, q + "downsample.0.weight", q + "downsample.1", stride, 0))
                descs.append(_conv_entry(sd, keep, q + "conv3.weight", q + "bn3", 1, 0))
            else:
                descs.append(_conv_entry(sd, keep, q + "conv1.weight", q + "bn1", stride, 1))
                if has_ds:
                    descs.append(_conv_entry(sd, keep, q + "downsample.0.weight", q + "downsample.1", stride, 0))
                descs.append(_conv_entry(sd, keep, q + "conv2.weight", q + "bn2", 1, 1))
    h = head_prefix
    if not head:
        return descs, keep
    if block == "bottleneck":
        descs.append(_conv_entry(sd, keep, h + "0.weight", None, 1, 1))
    else:
        descs.append(_conv_entry(sd, keep, h + "0.conv1.weight", h + "0.bn1", 1, 1))
        descs.append(_conv_entry(sd, keep, h + "0.conv2.weight", h + "0.bn2", 1, 1))
        descs.append(_conv_entry(sd, keep, h + "1.weight", None, 1, 1))
    return descs, keep


class BackboneEngine:
    """Owns a `b200trk_net_t`. forward(im) mirrors NetWithBackbone.extract_backbone + extract_classification_feat.
    `precision`: 0 = 3xTF32 on the tensor cores (fp32-faithful), 1 = exact fp32 on the CUDA cores, 2 = single-pass TF32 on the tensor
    cores (each operand rounded once to TF32, fp32 accumulation: the numerics cuDNN gives a PyTorch convolution with TF32 allowed).
    The precision covers every convolution of the plan, the heads attached later included."""

    def __init__(self, state_dict, arch="resnet50", filter_size=4, max_batch=1, crop_size=288, precision=0, device=None, head=True,
                 head_prefix="classifier.feature_extractor.", norm_scale=None):
        if not torch.cuda.is_available():
            raise RuntimeError("BackboneEngine: CUDA device required (the engine has no CPU path)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.arch = arch
        self.max_batch = max_batch
        self.crop_size = (crop_size, crop_size) if isinstance(crop_size, int) else tuple(crop_size)
        descs, keep = conv_descs_from_state_dict(state_dict, arch, head=head, head_prefix=head_prefix)
        self.has_head = head
        arr = (_lib.ConvDesc * len(descs))(*descs)
        out_dim = descs[-1].cout
        # InstanceL2Norm scale: sqrt(1 / (out_dim * filter_size^2)) (dimpnet.py:159, tompnet.py:131) unless given explicitly
        self.norm_scale = math.sqrt(1.0 / (out_dim * filter_size * filter_size)) if norm_scale is None else float(norm_scale)
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_net_create(C.byref(handle), ARCH_ID[arch], arr, len(descs), self.norm_scale,
                                                     max_batch, self.crop_size[0], self.crop_size[1], precision), "net_create")
        del keep
        self.handle = handle
        dims = (C.c_int * 9)()
        _lib.check(_lib.lib().b200trk_net_dims(self.handle, C.byref(dims)), "net_dims")
        self.dims = list(dims)
        self.flops = _lib.lib().b200trk_net_flops(self.handle)

    def attach_iou_head(self, state_dict, prefix="bb_regressor."):
        """Append AtomIoUNet.get_iou_feat (atom_iou_net.py:172-179) to the plan; forward(want=(..., 'iou3', 'iou4')) then also
        returns the two IoU feature maps."""
        keep, descs = [], []
        for name in ("conv3_1t", "conv3_2t", "conv4_1t", "conv4_2t"):
            q = prefix + name
            descs.append(_conv_entry(state_dict, keep, q + ".0.weight", q + ".1", 1, 1, bias_key=q + ".0.bias"))
        arr = (_lib.ConvDesc * 4)(*descs)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_net_attach_iou_head(self.handle, arr), "net_attach_iou_head")
        d = (C.c_int * 6)()
        _lib.check(_lib.lib().b200trk_net_iou_dims(self.handle, C.byref(d)), "net_iou_dims")
        self.iou_dims = list(d)
        self.flops = _lib.lib().b200trk_net_flops(self.handle)
        del keep

    def attach_iou_ref(self, state_dict, prefix="bb_regressor."):
        """AtomIoUNet's conv3_1r / conv4_1r (atom_iou_net.py:30-35) as plan steps for get_modulation (iou.IoUModulation)."""
        keep, descs = [], []
        for name in ("conv3_1r", "conv4_1r"):
            q = prefix + name
            descs.append(_conv_entry(state_dict, keep, q + ".0.weight", q + ".1", 1, 1, bias_key=q + ".0.bias"))
        arr = (_lib.ConvDesc * 2)(*descs)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_net_attach_iou_ref(self.handle, arr), "net_attach_iou_ref")
        self.has_iou_ref = True
        del keep

    def attach_filter_init(self, state_dict, filter_size=4, filter_norm=False, pool_square=False,
                           prefix="classifier.filter_initializer."):
        """FilterInitializerLinear (initializer.py:118-173) from the state_dict's filter_conv; `filter_norm` / `pool_square` are its
        constructor arguments (init_filter_norm / init_pool_square of dimpnet50 / klcedimpnet50, both False there)."""
        keep = []
        d = _conv_entry(state_dict, keep, prefix + "filter_conv.weight", None, 1, state_dict[prefix + "filter_conv.weight"].shape[-1] // 2,
                        bias_key=prefix + "filter_conv.bias")
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().b200trk_net_attach_filter_init(self.handle, C.byref(d), int(filter_size), int(bool(filter_norm)),
                                                                 int(bool(pool_square))), "net_attach_filter_init")
        self.filter_size = int(filter_size)
        del keep

    def filter_init(self, clf, boxes, images=None):
        """FilterInitializerLinear.forward: clf [S,C,H,W] normalised classification features (CUDA), boxes [n,4] (x, y, w, h), box r on
        image images[r] (default r) -> filter [1,C,k,k], the mean over the n boxes."""
        clf = clf.contiguous()
        b = torch.as_tensor(boxes, dtype=torch.float32).reshape(-1, 4).contiguous().cpu()
        img = None if images is None else (C.c_int * b.shape[0])(*[int(i) for i in images])
        k = self.filter_size
        out = torch.empty(1, clf.shape[1], k, k, device=clf.device, dtype=torch.float32)
        _lib.check(_lib.lib().b200trk_net_filter_init(self.handle, C.c_void_p(clf.data_ptr()), int(clf.shape[0]), int(b.shape[0]),
                                                      img, C.c_void_p(b.data_ptr()), C.c_void_p(out.data_ptr()),
                                                      C.c_void_p(torch.cuda.current_stream(clf.device).cuda_stream)), "net_filter_init")
        return out

    def iou_features(self, s):
        """get_iou_feat on the activations of the last forward pass (batch s) still in the arena -> (iou3, iou4)."""
        dev = self.device
        i3 = torch.empty(s, *self.iou_dims[0:3], device=dev, dtype=torch.float32)
        i4 = torch.empty(s, *self.iou_dims[3:6], device=dev, dtype=torch.float32)
        _lib.check(_lib.lib().b200trk_net_iou_from_arena(self.handle, s, C.c_void_p(i3.data_ptr()), C.c_void_p(i4.data_ptr()),
                                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)), "net_iou_from_arena")
        return i3, i4

    def forward(self, im, want=("layer2", "layer3", "classification")):
        """im: [S,3,H,W] CUDA float32 in pixel range 0..255. Returns OrderedDict of NCHW CUDA tensors."""
        if not im.is_cuda or im.dtype != torch.float32:
            raise RuntimeError("BackboneEngine.forward: input must be a CUDA float32 tensor")
        im = im.contiguous()
        s = im.shape[0]
        if tuple(im.shape[1:]) != (3,) + self.crop_size:
            raise RuntimeError("BackboneEngine.forward: expected [S,3,%d,%d], got %s" % (self.crop_size + (tuple(im.shape),)))
        d = self.dims
        outs = OrderedDict()
        ptrs = []
        for i, name in enumerate(("layer2", "layer3", "classification")):
            if name in want and (name != "classification" or self.has_head):
                t = torch.empty(s, d[3 * i], d[3 * i + 1], d[3 * i + 2], device=im.device, dtype=torch.float32)
                outs[name] = t
                ptrs.append(C.c_void_p(t.data_ptr()))
            else:
                ptrs.append(C.c_void_p(0))
        for i, name in enumerate(("iou3", "iou4")):
            if name in want:
                if not getattr(self, "iou_dims", None):
                    raise RuntimeError("BackboneEngine.forward: '%s' requested but no IoU head is attached" % name)
                t = torch.empty(s, *self.iou_dims[3 * i:3 * i + 3], device=im.device, dtype=torch.float32)
                outs[name] = t
                ptrs.append(C.c_void_p(t.data_ptr()))
            else:
                ptrs.append(C.c_void_p(0))
        _lib.check(_lib.lib().b200trk_net_forward_iou(self.handle, C.c_void_p(im.data_ptr()), s, ptrs[0], ptrs[1], ptrs[2], ptrs[3],
                                                      ptrs[4], C.c_void_p(torch.cuda.current_stream().cuda_stream)), "net_forward")
        return outs

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle:
            _lib.lib().b200trk_net_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
