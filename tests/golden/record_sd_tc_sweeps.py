"""Records tests/golden/sd_tc_sweeps.npz: the filters of the tensor-core steepest-descent kernel on the seeded cases of
tests/test_sd_tc_sweeps_gpu.py. Run on an H100 from the repository root after build():

    python tests/golden/record_sd_tc_sweeps.py [OUT.npz]

The recording pins the kernel's output bit for bit, so it is taken from a build whose output is the accepted one."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from pytracking_b200 import _lib  # noqa: E402
from test_sd_tc_sweeps_gpu import CASES, case_key, run_case  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "sd_tc_sweeps.npz")
    os.environ.pop("B200TRK_SD_TC", None)
    rec = {}
    for kind, n in CASES:
        rec[case_key(kind, n)] = run_case(kind, n)
        assert _lib.lib().b200trk_sd_last_kernel() == 1
    np.savez_compressed(out, **rec)
    print("recorded %d filters on %s -> %s" % (len(rec), torch.cuda.get_device_name(0), out))


if __name__ == "__main__":
    main()
