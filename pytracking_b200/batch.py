"""Several DiMP / PrDiMP sequences tracked in lock-step on one GPU (`b200trk_dimp_batch_*`, include/b200trk.h).

A `DiMPBatchTracker` of capacity S holds S slots on one network built for batches of S.  One `step()` takes a frame for any subset of
the slots and runs one crop launch, one network forward at batch S, one classify and one localisation launch for all of them, then
each slot's host update and its own online filter update.  The forward always runs at batch S, so a sequence's boxes depend only on
its own frames and on S -- not on which other sequences share the batch or when they started.  `track_sequences` runs a dataset of
sequences through it, starting the next sequence in a slot as soon as the previous one ends."""
import ctypes as C
import time

import numpy as np
import torch

from . import _lib
from .engine import BackboneEngine
from .frame_engine import _view, optimizer_args
from .tracker import frame_pointer, tracker_settings


class DiMPBatchTracker:
    """`state_dict`, `params`, `arch`, `newton` as for `DiMPTracker` (newton=None: DiMP's GN optimiser; a dict: PrDiMP's Newton
    optimiser, whose softmax_reg the localisation then uses).  use_iou_net must be False."""

    def __init__(self, state_dict, params, capacity, arch="resnet50", newton=None, device=None, precision=0, **param_overrides):
        self.params, newton = tracker_settings(params, newton, **param_overrides)
        p = self.params
        if p.use_iou_net:
            raise RuntimeError("DiMPBatchTracker: use_iou_net is not supported in a batch; set use_iou_net=False")
        if not 1 <= int(capacity) <= 16:
            raise RuntimeError("DiMPBatchTracker: capacity=%r outside 1..16" % (capacity,))
        self.capacity = int(capacity)
        self.backbone = BackboneEngine(state_dict, arch, 4, self.capacity, p.image_sample_size, precision, device)
        self.device = self.backbone.device
        args, _, _ = optimizer_args(state_dict, newton)
        create = "dimp_batch_create" if newton is None else "prdimp_batch_create"
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(getattr(_lib.lib(), "b200trk_" + create)(C.byref(h), self.backbone.handle, self.capacity, C.byref(p), 4, *args),
                       create)
        self.handle = h
        cc, hc, wc = self.backbone.dims[6:9]
        self.feat_dims = (cc, hc, wc)
        self.out_sz = (hc + 1, wc + 1)
        self._items = (_lib.BatchItem * self.capacity)()
        self._infos = (_lib.FrameInfo * self.capacity)()
        self._pinned = {}
        self.last_info = {}

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def step(self, frames):
        """frames: {slot: (frame, init_info_or_None)}.  init_info = {'init_bbox': [x, y, w, h]} starts a sequence in the slot; None
        tracks the slot's running sequence.  Frames are uint8 [H,W,3] host arrays, or all CUDA tensors (kept in HBM: no upload).
        Returns {slot: {'target_bbox': [x, y, w, h]}} (for an init frame, the init box)."""
        if not frames:
            return {}
        if len(frames) > self.capacity:
            raise RuntimeError("DiMPBatchTracker.step: %d frames for %d slots" % (len(frames), self.capacity))
        keep, slots = [], []
        on_device = None
        for k, (slot, (frame, init)) in enumerate(frames.items()):
            it = self._items[k]
            buf, ptr, H, W, dev = frame_pointer(frame, self._pinned, slot, "DiMPBatchTracker.step")
            keep.append(buf)
            if on_device is None:
                on_device = dev
            elif on_device != dev:
                raise RuntimeError("DiMPBatchTracker.step: all frames of a step must be on the host or all on the GPU")
            it.slot, it.image, it.H, it.W = int(slot), ptr, int(H), int(W)
            it.init = int(init is not None)
            for i in range(4):
                it.init_bbox[i] = float(init["init_bbox"][i]) if init is not None else 0.0
            slots.append(int(slot))
        fn = _lib.lib().b200trk_dimp_batch_step_device if on_device else _lib.lib().b200trk_dimp_batch_step_host
        with torch.cuda.device(self.device):
            _lib.check(fn(self.handle, self._items, len(slots), self._infos, self._stream()), "dimp_batch_step")
        out = {}
        for k, slot in enumerate(slots):
            info = self._infos[k]
            self.last_info[slot] = info
            out[slot] = {"target_bbox": [float(v) for v in info.bbox]}
        return out

    def release(self, slot):
        _lib.check(_lib.lib().b200trk_dimp_batch_release(self.handle, int(slot)), "dimp_batch_release")

    # ---- read-only views of one slot (device memory owned by the library) ----------------------------------------------------
    def filter(self, slot):
        cc = self.feat_dims[0]
        return _view(_lib.lib().b200trk_dimp_batch_filter(self.handle, int(slot)), (1, cc, 4, 4), self, self.device)

    def scores(self, slot):
        return _view(_lib.lib().b200trk_dimp_batch_scores(self.handle, int(slot)), self.out_sz, self, self.device)

    def crop(self, slot):
        iss = self.params.image_sample_size
        return _view(_lib.lib().b200trk_dimp_batch_crop(self.handle, int(slot)), (3, iss, iss), self, self.device)

    def state(self, slot):
        out = (C.c_float * 9)()
        _lib.check(_lib.lib().b200trk_dimp_batch_state(self.handle, int(slot), C.byref(out)), "dimp_batch_state")
        return np.array(out, dtype=np.float32)

    def close(self):
        if getattr(self, "handle", None):
            _lib.lib().b200trk_dimp_batch_destroy(self.handle)
            self.handle = None
        if getattr(self, "backbone", None) is not None:
            self.backbone.close()
            self.backbone = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def track_sequences(tracker, sequences):
    """Track every `(frames, init_bbox)` of `sequences` (frames: any iterable of uint8 [H,W,3] frames, the first one the init frame)
    on a DiMPBatchTracker, keeping every slot busy: when a sequence ends its slot starts the next waiting sequence in the same step.
    Returns, per sequence in input order, {'target_bbox': [box per frame], 'time': [seconds per frame]} -- the shape of the
    reference's run_sequence output (frame 0 carries the init box).  A frame's time is the wall time of the step that tracked it."""
    pending = list(enumerate(sequences))[::-1]
    results = [None] * len(pending)
    running = {}                                  # slot -> (sequence index, frame iterator)

    def start(slot):
        q, (frames, init_bbox) = pending.pop()
        results[q] = {"target_bbox": [], "time": []}
        running[slot] = (q, iter(frames), [float(v) for v in init_bbox])

    for slot in range(tracker.capacity):
        if pending:
            start(slot)
    first = set(running)
    while running:
        batch = {}
        for slot in list(running):
            q, it, init_bbox = running[slot]
            frame = next(it, None)
            if frame is None:                     # sequence finished: hand the slot to the next one
                del running[slot]
                tracker.release(slot)
                if pending:
                    start(slot)
                    first.add(slot)
                    q, it, init_bbox = running[slot]
                    frame = next(it, None)
                if frame is None:
                    continue
            batch[slot] = (frame, {"init_bbox": init_bbox} if slot in first else None)
        first.clear()
        if not batch:
            continue
        t0 = time.perf_counter()
        out = tracker.step(batch)
        dt = time.perf_counter() - t0
        for slot, o in out.items():
            r = results[running[slot][0]]
            r["target_bbox"].append(o["target_bbox"])
            r["time"].append(dt)
    return results
