"""The three kernels of a batch step (csrc/dimp_tracker_kernels.cuh: sample_patch_batch_kernel, classify_batch_kernel,
localize_batch_kernel) executed ON THE CPU under tests/cpu_emul/cuda_shim.h (tests/cpu_emul/batch_emul.cpp), against the single-sequence
kernels a solo tracker runs and against torch-CPU bilinear resampling:
  * one batched crop launch over items mixing the nine sampler geometries of test_dimp_kernels_cpu, two frame sizes and the windowed
    first-frame crop is bit-exact with the reference's sample_patch resampled by torch on the CPU, item for item;
  * the batched localisation gives, item for item, the bytes of localize_kernel on the score maps of the recorded reference trajectories
    (DiMP, and PrDiMP with the softmax pre-processing), slots in shuffled order;
  * the per-slot classify equals a single-sample apply_filter_kernel with that slot's filter, bit for bit.
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from pytracking_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp("batch_emul")), "libbatch_emul.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    os.path.join(ROOT, "tests", "cpu_emul", "batch_emul.cpp"), "-o", out], check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.batch_emul_classify.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_int, C.c_int]
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def test_batched_sampler_bit_exact_vs_torch_cpu(emul):
    from oracle import preprocessing_ref as R
    from pytracking_b200.tracker import HostLogic, make_params
    from tracker_cases import DIMP50
    rng = np.random.RandomState(5)
    cases = [(480, 640, [300, 200, 80, 60]), (480, 640, [2, 3, 90, 70]), (480, 640, [600, 440, 80, 60]), (720, 1280, [500, 300, 400, 300]),
             (1080, 1920, [1500, 900, 410, 170]), (240, 320, [150, 100, 9, 9]), (480, 640, [100, 100, 3, 2]),
             (2160, 3840, [1000, 1000, 1500, 900]), (300, 300, [100, 100, 57.6, 57.6])]
    imgs, geoms, refs = [], [], []
    for k, (H, W, bb) in enumerate(cases):
        img = np.ascontiguousarray(rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
        hl = HostLogic(make_params(**dict(DIMP50, augmentation_expansion_factor=2 if k in (0, 4) else None)))
        g_init, _ = hl.init_state(H, W, bb)
        st = hl.state()
        im = R.numpy_to_torch(img)
        sz = torch.tensor([288.0, 288.0])
        if k in (0, 4):                          # the windowed first-frame crop (expanded 576^2 patch, 288^2 window)
            g = g_init
            ref = R.sample_init_patch(im, torch.tensor([st[0], st[1]]).round(), torch.tensor(st[4]), sz, 2)
            assert g.out_h == 576 and g.win_r == 144
        else:
            g = hl.plan_crop()
            ref, _ = R.sample_patch(im, torch.tensor([st[0], st[1]]), torch.tensor(st[4]) * sz, sz)
        hl.close()
        imgs.append(img); geoms.append(g); refs.append(ref[0])
    n = len(cases)
    dst = np.array(np.random.RandomState(1).permutation(16)[:n], np.int32)          # items land in shuffled slots of a capacity-16 buffer
    out = np.full((16, 3, 288, 288), np.nan, np.float32)
    ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
    Hs, Ws = np.array([c[0] for c in cases], np.int32), np.array([c[1] for c in cases], np.int32)
    gs = (_lib.CropGeom * n)(*geoms)
    assert emul.batch_emul_sample_patch(ptrs, _ptr(Hs), _ptr(Ws), gs, _ptr(dst), n, 288, _ptr(out)) == 0
    for k in range(n):
        assert torch.equal(torch.from_numpy(out[dst[k]]), refs[k]), (k, cases[k])
        single = np.empty((3, 288, 288), np.float32)
        assert emul.batch_emul_sample_patch_single(_ptr(imgs[k]), int(Hs[k]), int(Ws[k]), C.byref(geoms[k]), 288, _ptr(single)) == 0
        assert np.array_equal(single.view(np.uint32), out[dst[k]].view(np.uint32)), k
    untouched = np.setdiff1d(np.arange(16), dst)
    assert np.isnan(out[untouched]).all()                                          # nothing outside the items' crops is written


def _trajectory_problems(kind):
    """(params, [(scores [Ho,Wo], neigh [2], prev_vec [2], recorded flag)]) replayed through the host logic as the tracker feeds them."""
    from pytracking_b200.tracker import HostLogic, make_params
    from tracker_cases import DIMP50, OVERRIDES, _loc
    if kind == "dimp":
        names, load, mk, fs, iss = ("cfg2", "stress"), "dimp_host_%s.npz", lambda nm: make_params(**dict(DIMP50, **OVERRIDES[nm])), 18, 288
    else:
        from test_prdimp_host_logic_cpu import prdimp_params
        names, load, mk, fs, iss = ("noaug", "stress"), "prdimp_host_%s.npz", prdimp_params, 22, 352
    out = []
    for name in names:
        d = np.load(os.path.join(GOLDEN, load % name))
        params = mk(name)
        hl = HostLogic(params)
        H, W = [int(v) for v in d["image_hw"]]
        hl.adopt(H, W, d["init_state"], d["init_sw"], d["init_counts"][0], d["init_counts"][1])
        for t in range(len(d["flag"])):
            g = hl.plan_crop()
            st = hl.state()
            neigh = [np.float32(np.float32(params.target_neighborhood_scale) * (st[2 + i] / np.float32(g.sample_scale))) * np.float32(fs / iss)
                     for i in range(2)]
            pv = [(st[i] - np.float32(g.sample_pos[i])) / (np.float32(16.0) * np.float32(g.sample_scale)) for i in range(2)]
            out.append((params, d["scores"][t].astype(np.float32), neigh, pv, int(d["flag"][t])))
            hl.commit(g, _loc(d, t))
        hl.close()
    return out


@pytest.mark.parametrize("kind", ["dimp", "prdimp"])
def test_batched_localisation_equals_single_kernel_on_recorded_trajectories(emul, kind):
    probs = _trajectory_problems(kind)
    rng = np.random.RandomState(7)
    flags, agree = set(), 0
    groups = [[c for c in probs if c[0] is p] for p in {id(c[0]): c[0] for c in probs}.values()]    # one parameter set per launch
    for group in groups:
        for start in range(0, len(group), 11):
            chunk = group[start:start + 11]
            params = chunk[0][0]
            n = len(chunk)
            ho, wo = chunk[0][1].shape
            slots = np.array(rng.permutation(16)[:n], np.int32)
            scores = np.ascontiguousarray(rng.rand(16, ho, wo).astype(np.float32))
            for i, c in enumerate(chunk):
                scores[slots[i]] = c[1]
            neigh = np.ascontiguousarray([c[2] for c in chunk], np.float32)
            pv = np.ascontiguousarray([c[3] for c in chunk], np.float32)
            res = (_lib.LocResult * n)()
            assert emul.batch_emul_localize(_ptr(scores), ho, wo, C.byref(params), _ptr(slots), _ptr(neigh), _ptr(pv), n, res) == 0
            for i, c in enumerate(chunk):
                one = _lib.LocResult()
                m = np.ascontiguousarray(c[1][None])
                assert emul.batch_emul_localize_single(_ptr(m), ho, wo, C.byref(params), _ptr(neigh[i]), _ptr(pv[i]), C.byref(one)) == 0
                assert bytes(res[i]) == bytes(one), (kind, start + i, res[i].flag, one.flag)
                flags.add(int(one.flag))
                agree += int(one.flag == c[4])
    assert flags >= {1, 2, 3}, flags
    assert agree >= len(probs) - 2                                   # the single kernel's own agreement with the recordings


@pytest.mark.parametrize("fs,c", [(18, 128), (22, 64)])
def test_per_slot_classify_equals_single_sample_apply_filter(emul, fs, c):
    from pytracking_b200 import synth
    n = 5
    feat = np.ascontiguousarray(synth.make_clf_features(11 + fs, n, c=c, h=fs, w=fs).numpy())
    g = torch.Generator().manual_seed(fs)
    stride = c * 16 + 48                                             # the filter stride is a parameter: not necessarily C*k*k
    filt = np.zeros(n * stride, np.float32)
    for i in range(n):
        filt[i * stride:i * stride + c * 16] = (torch.randn(c * 16, generator=g) * 0.05).numpy()
    scores = np.full((n, fs + 1, fs + 1), np.nan, np.float32)
    assert emul.batch_emul_classify(_ptr(feat), _ptr(filt), stride, _ptr(scores), n, c, fs) == 0
    for i in range(n):
        one = np.empty((fs + 1, fs + 1), np.float32)
        f = np.ascontiguousarray(filt[i * stride:i * stride + c * 16])
        assert emul.batch_emul_apply_filter_single(_ptr(np.ascontiguousarray(feat[i])), _ptr(f), _ptr(one), c, fs) == 0
        assert np.array_equal(one.view(np.uint32), scores[i].view(np.uint32)), i
