"""CPU tier of the first-frame augmentation (csrc/augment_kernels.cuh, b200trk_dimp_tracker_init_state_augmented), against
tests/golden/augment.npz (oracle/gen_augment_golden.py: the unmodified reference with cv2) and oracle/augmentation_ref.py:
  * the oracle's rotation equals cv2.warpAffine bit for bit; its identity, translation, flip and rotate crops of the expanded patch
    equal the reference's 13 crops (SHA-256) bit for bit; its tap-order blur and the reference's blurred crops lie within the float32
    bound of a float64 convolution;
  * the kernel sources under tests/cpu_emul/cuda_shim.h: translation, flip and rotate bit for bit with the oracle, the blur bit for bit
    with the oracle's tap-order sums and within the float64 bound -- at 576 -> 288, 704 -> 352, expansion factor 1, and with shifts
    that push the window past the patch; clean under ThreadSanitizer and AddressSanitizer (exact-size dynamic shared memory) with the
    alignment check;
  * the host half: draws from torch's CPU generator give the reference's shifts and dropout masks, the 15 target boxes and the
    scalar state are the golden's bit for bit, and the augmented start replays the recorded dimp_host_cfg2 / dimp_host_stress
    trajectories (recorded with augmentation); refusals leave the tracker as it was."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import augmentation_ref as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "augment.npz")
SRC = os.path.join(ROOT, "tests", "cpu_emul", "augment_emul.cpp")
STOCK = {"fliplr": True, "rotate": [10, -10, 45, -45], "blur": [(3, 1), (1, 3), (2, 2)],
         "relativeshift": [(0.6, 0.6), (-0.6, 0.6), (0.6, -0.6), (-0.6, -0.6)], "dropout": (2, 0.2)}
PARAMS = {"dimp_": 0, "prdimp_": 1}          # prefix -> synth.make_sequence index of the recorded first frame


def golden():
    return np.load(GOLDEN)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def params(prefix):
    from pytracking_b200.tracker import make_params
    if prefix == "dimp_":
        from tracker_cases import DIMP50
        return make_params(**DIMP50)
    from test_prdimp_host_logic_cpu import prdimp_params
    return prdimp_params()


def stock_list(d, prefix):
    """(kind, shift, param) of the recorded transforms, parameters from the stock dict in generate_init_samples' order."""
    par = [None] * 5 + [None] + list(STOCK["blur"]) + list(STOCK["rotate"])
    return [(int(k), tuple(int(v) for v in s), p) for k, s, p in zip(d[prefix + "kinds"], d[prefix + "shifts"], par)]


def expanded_patch(prefix, d):
    """The reference's expanded first-frame patch (sample_patch at the expansion size), restated by oracle/preprocessing_ref.py."""
    from oracle import preprocessing_ref as R
    from pytracking_b200 import synth
    frames, _ = synth.make_sequence(PARAMS[prefix], num_frames=1)
    st = d[prefix + "init_state"]
    iss = 288 if prefix == "dimp_" else 352
    big = torch.tensor([2.0 * iss, 2.0 * iss])
    pos = torch.tensor([st[0], st[1]]).round()
    patch, _ = R.sample_patch(R.numpy_to_torch(frames[0]), pos, torch.tensor(st[4]) * big, big)
    return np.ascontiguousarray(patch[0].numpy()), iss


def test_oracle_rotation_is_cv2_bit_for_bit():
    from oracle.gen_augment_golden import WARP_ANGLES, WARP_SIZES, STOCK_ANGLES, warp_image
    d = golden()
    for h, w in WARP_SIZES:
        img = warp_image(h, w, h * 100 + w).transpose(2, 0, 1).copy()
        for i, a in enumerate(WARP_ANGLES):
            assert np.array_equal(A.rotate(img, a).transpose(1, 2, 0), d["warp_%dx%d_%d" % (h, w, i)]), (h, w, a)
    big = warp_image(576, 576, 576).transpose(2, 0, 1).copy()
    for a, dg in zip(STOCK_ANGLES, d["warp576_digest"]):
        assert digest(A.rotate(big, a).transpose(1, 2, 0)) == str(dg), a


@pytest.mark.parametrize("prefix", list(PARAMS))
def test_oracle_crops_are_the_reference_crops(prefix):
    d = golden()
    patch, iss = expanded_patch(prefix, d)
    blur_i = 0
    for k, (kind, shift, par) in enumerate(stock_list(d, prefix)):
        out = A.transform(patch, kind, shift, par, (iss, iss))
        if kind != 3:
            assert digest(out) == str(d[prefix + "crop_digest"][k]), (prefix, k, kind)
            continue
        # the reference's blur (torch conv2d) and the oracle's tap-order sum, both against float64
        ref64 = A.crop(A.blur64(patch, par), (iss, iss), shift)
        bound = A.blur_bound(patch, par)
        assert np.abs(out.astype(np.float64) - ref64).max() <= bound, (prefix, k)
        w = d[prefix + "blur_window"][blur_i]
        from oracle.gen_augment_golden import CROP_WINDOW
        assert np.abs(w.astype(np.float64) - ref64[CROP_WINDOW]).max() <= bound, (prefix, k)
        blur_i += 1


def _build(out, flags=()):
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique",
                    "-Wno-unknown-pragmas"] + list(flags) + [SRC, "-o", out], check=True, capture_output=True)
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    return C.CDLL(_build(os.path.join(str(tmp_path_factory.mktemp("augment_emul")), "libaugment_emul.so")))


def descriptor(xf):
    from pytracking_b200 import _lib
    arr = (_lib.AugTransform * len(xf))()
    for k, (kind, shift, par) in enumerate(xf):
        arr[k].kind, arr[k].shift[0], arr[k].shift[1] = kind, int(shift[0]), int(shift[1])
        p = (0.0, 0.0) if par is None else ((float(par), 0.0) if np.isscalar(par) else tuple(float(v) for v in par))
        arr[k].param[0], arr[k].param[1] = p
    return arr


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def run_emul(emul, patch, out_hw, xf):
    crops = np.full((len(xf), 3) + tuple(out_hw), np.nan, np.float32)
    rc = emul.aug_emul_crops(_p(patch), patch.shape[1], patch.shape[2], out_hw[0], out_hw[1], descriptor(xf), len(xf), _p(crops))
    return rc, crops


def check_against_oracle(crops, patch, xf, out_hw, where):
    for k, (kind, shift, par) in enumerate(xf):
        ref = A.transform(patch, kind, shift, par, out_hw)
        assert np.array_equal(crops[k], ref), (where, k, kind, shift, float(np.abs(crops[k] - ref).max()))
        if kind == 3:
            e = np.abs(crops[k].astype(np.float64) - A.crop(A.blur64(patch, par), out_hw, shift)).max()
            assert e <= A.blur_bound(patch, par), (where, k, e)


def random_patch(seed, h, w):
    return (np.random.RandomState(seed).rand(3, h, w) * 255).astype(np.float32)


@pytest.mark.parametrize("prefix", list(PARAMS))
def test_kernel_sources_match_oracle_on_the_recorded_first_frames(emul, prefix):
    d = golden()
    patch, iss = expanded_patch(prefix, d)
    xf = stock_list(d, prefix)
    rc, crops = run_emul(emul, patch, (iss, iss), xf)
    assert rc == 0
    check_against_oracle(crops, patch, xf, (iss, iss), prefix)
    for k, (kind, _, _) in enumerate(xf):
        if kind != 3:
            assert digest(crops[k]) == str(d[prefix + "crop_digest"][k]), (prefix, k)


# shifts that push the window past the patch (clamped indices), expansion factor 1, non-square patches
EDGE_CASES = [
    ((100, 100), (50, 50), [(0, (0, 0), None), (1, (60, -70), None), (2, (-40, 45), None), (3, (55, -30), (3, 1)), (4, (-50, 52), 45),
                            (4, (30, 0), -10), (3, (-48, 60), (1.5, 2.5))]),
    ((64, 64), (64, 64), [(0, (0, 0), None), (1, (9, -7), None), (2, (3, 4), None), (3, (-5, 6), (2, 2)), (4, (7, -8), 10)]),
    ((90, 70), (40, 36), [(0, (0, 0), None), (1, (-200, 230), None), (2, (180, -170), None), (3, (160, -150), (1, 3)), (4, (190, 200), -45),
                          (4, (0, 0), 30)]),
]


@pytest.mark.parametrize("case", range(len(EDGE_CASES)))
def test_kernel_sources_clamp_and_other_geometries(emul, case):
    in_hw, out_hw, xf = EDGE_CASES[case]
    patch = random_patch(10 + case, *in_hw)
    rc, crops = run_emul(emul, patch, out_hw, xf)
    assert rc == 0
    check_against_oracle(crops, patch, xf, out_hw, case)


def test_kernel_sources_refuse_scale_and_wide_blur(emul):
    patch = random_patch(0, 40, 40)
    assert run_emul(emul, patch, (20, 20), [(0, (0, 0), None), (5, (0, 0), 1.05)])[0] == 2
    assert run_emul(emul, patch, (20, 20), [(0, (0, 0), None), (3, (0, 0), (9.0, 1.0))])[0] == 2


def test_dropout_kernel_source(emul):
    rng = np.random.RandomState(3)
    T, num, Cc, HW = 3, 2, 40, 18 * 18
    clf = rng.randn(T + num, Cc, HW).astype(np.float32)
    mult = (rng.rand(num, Cc) > 0.2).astype(np.float32) * np.float32(1.25)
    out = clf.copy()
    assert emul.aug_emul_dropout(_p(out), T, num, Cc, HW, _p(mult)) == 0
    assert np.array_equal(out[:T], clf[:T])
    assert np.array_equal(out[T:], (torch.from_numpy(clf[0:1]).expand(num, Cc, HW) * torch.from_numpy(mult)[:, :, None]).numpy())


_SWEEP = r"""
import ctypes as C, sys
import numpy as np
L = C.CDLL(sys.argv[1])
sys.path.insert(0, sys.argv[2])
from pytracking_b200 import _lib
P = lambda a: a.ctypes.data_as(C.c_void_p)
rng = np.random.RandomState(0)
patch = np.ascontiguousarray((rng.rand(3, 70, 60) * 255).astype(np.float32))
xf = [(0, (0, 0), (0, 0)), (1, (30, -40), (0, 0)), (2, (-5, 3), (0, 0)), (3, (50, -45), (3.0, 1.0)), (3, (0, 0), (8.0, 8.0)), (4, (10, 60), (45.0, 0))]
arr = (_lib.AugTransform * len(xf))()
for k, (kind, s, p) in enumerate(xf):
    arr[k].kind, arr[k].shift[0], arr[k].shift[1] = kind, s[0], s[1]
    arr[k].param[0], arr[k].param[1] = p
crops = np.zeros((len(xf), 3, 40, 40), np.float32)
assert L.aug_emul_crops(P(patch), 70, 60, 40, 40, arr, len(xf), P(crops)) == 0
clf, mult = np.ascontiguousarray(rng.randn(4, 8, 9).astype(np.float32)), np.ones((2, 8), np.float32)
L.aug_emul_dropout(P(clf), 2, 2, 8, 9, P(mult))
print("EMUL_DONE")
"""


@pytest.mark.parametrize("sanitizer", ["thread", "address"])
def test_kernel_sources_under_sanitizers(tmp_path, sanitizer):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    rt = subprocess.run(["g++", "-print-file-name=lib%s.so" % ("tsan" if sanitizer == "thread" else "asan")], capture_output=True,
                        text=True).stdout.strip()
    if not os.path.isabs(rt) or not os.path.exists(rt):
        pytest.skip("no %s sanitizer runtime" % sanitizer)
    flags = ["-fsanitize=%s,alignment" % sanitizer] + (["-Wno-tsan"] if sanitizer == "thread" else [])
    lib = _build(str(tmp_path / ("libaugment_%s.so" % sanitizer)), flags)
    env = dict(os.environ, LD_PRELOAD=rt, B200_EMUL_THREADS="1",
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-c", _SWEEP, lib, ROOT], capture_output=True, text=True, env=env, timeout=900)
    if "EMUL_DONE" not in r.stdout and "Sanitizer" not in r.stderr:
        pytest.skip("the %s sanitizer could not run here: %s" % (sanitizer, r.stderr[-300:]))
    assert "EMUL_DONE" in r.stdout, r.stderr[-3000:]
    for bad in ("data race", "runtime error", "AddressSanitizer"):
        assert bad not in r.stderr, r.stderr[:4000]


def draw(seed=0):
    from pytracking_b200.tracker import draw_augmentation
    torch.manual_seed(seed)
    return draw_augmentation(STOCK, 288, 1 / 3, 512)


@pytest.mark.parametrize("prefix", list(PARAMS))
def test_host_half_gives_the_reference_boxes_draws_and_state(prefix):
    from pytracking_b200 import synth
    from pytracking_b200.tracker import HostLogic, draw_augmentation
    d = golden()
    iss = 288 if prefix == "dimp_" else 352
    torch.manual_seed(0)
    desc, mult = draw_augmentation(STOCK, iss, 1 / 3, 512)
    T = desc.num_transforms
    assert [desc.transform[k].kind for k in range(T)] == list(d[prefix + "kinds"])
    assert [[desc.transform[k].shift[0], desc.transform[k].shift[1]] for k in range(T)] == d[prefix + "shifts"].tolist()
    assert np.array_equal(mult.numpy(), d[prefix + "dropout"])
    frames, bb = synth.make_sequence(PARAMS[prefix], num_frames=1)
    hl = HostLogic(params(prefix))
    g, boxes = hl.init_state_augmented(480, 640, bb, desc)
    assert np.array_equal(boxes, d[prefix + "boxes"])
    assert np.array_equal(hl.state(), d[prefix + "init_state"])
    assert (g.out_h, g.out_w) == (2 * iss, 2 * iss)
    hl.close()


@pytest.mark.parametrize("name", ["cfg2", "stress"])
def test_augmented_start_replays_the_recorded_augmented_trajectories(name):
    """dimp_host_cfg2 / dimp_host_stress were recorded with the stock augmentation: the augmented host half gives their initial
    state, weights and counts, and the trajectory that follows replays as the adopted state does (tests/test_tracker_host_logic_cpu.py)."""
    from pytracking_b200.tracker import HostLogic, make_params
    from tracker_cases import DIMP50, GOLDEN as GD, OVERRIDES, _loc
    d = np.load(os.path.join(GD, "dimp_host_%s.npz" % name))
    desc, _keep = draw()
    hl = HostLogic(make_params(**dict(DIMP50, **OVERRIDES[name])))
    H, W = [int(v) for v in d["image_hw"]]
    g, boxes = hl.init_state_augmented(H, W, d["init_bbox"], desc)
    assert np.array_equal(hl.state(), d["init_state"])
    assert np.array_equal(boxes[0], d["init_target_box"])
    assert np.array_equal(np.array(g.sample_pos), d["init_sample_pos"]) and np.float32(g.sample_scale) == d["init_sample_scale"]
    assert tuple(d["init_counts"]) == (15, 15) and len(boxes) == 15
    max_sw_err = 0.0
    for t in range(len(d["flag"])):
        g = hl.plan_crop()
        assert np.array_equal(np.array(g.coord, dtype=np.float32), d["coord"][t]), (name, t)
        info, sw = hl.commit(g, _loc(d, t))
        assert np.array_equal(np.array(info.bbox, dtype=np.float32), d["bbox"][t]), (name, t)
        assert info.updated == d["updated"][t] and info.num_iter == d["num_iter"][t], (name, t)
        if info.updated:
            assert info.replace_ind == d["replace_ind"][t], (name, t)
            max_sw_err = max(max_sw_err, float(np.abs(sw - d["sw"][t]).max() / d["sw"][t].max()))
        if info.num_iter:
            assert info.n_stored == d["n_stored"][t]
    assert max_sw_err < 2e-6, max_sw_err
    hl.close()


def test_host_half_refusals_change_nothing():
    from pytracking_b200 import _lib
    from pytracking_b200.tracker import HostLogic, make_params
    from tracker_cases import DIMP50
    hl = HostLogic(make_params(**DIMP50))
    hl.init_state(480, 640, [300, 200, 80, 60])
    before = hl.state().copy()

    def refused(mutate):
        desc, keep = draw()
        mutate(desc)
        with pytest.raises(RuntimeError):
            hl.init_state_augmented(480, 640, [10, 20, 30, 40], desc)
        assert np.array_equal(hl.state(), before)

    refused(lambda d: setattr(d.transform[3], "kind", _lib.AUG_KINDS["scale"]))
    refused(lambda d: setattr(d, "num_dropout", 4))                       # 13 + 4 samples
    refused(lambda d: setattr(d.transform[0], "kind", _lib.AUG_KINDS["fliplr"]))
    refused(lambda d: setattr(d.transform[6], "param", (C.c_double * 2)(9.0, 1.0)))
    inside = HostLogic(make_params(**dict(DIMP50, border_mode="inside")))
    desc, keep = draw()
    with pytest.raises(RuntimeError):
        inside.init_state_augmented(480, 640, [10, 20, 30, 40], desc)
    inside.close()
    hl.close()
