"""Shared-memory layout of the tensor-core steepest-descent kernel (pytracking_b200/csrc/sd_tc.cu): the adjoint sweep's R^T tiles.

Right after the residual, every CTA builds the B tile R^T (hi | lo, 4 KB) of each (sample, pixel block) pair its adjoint range
touches, once per iteration, into slot i mod (n * KBT) for unit t_lo + i; the consumers then walk the range with a running slot
counter.  The tiles share one region with F^T (kba tiles), and launch_sd_tc sizes it as max(kba, min(ceil(UT / G), n * KBT)) tiles.
The wgmma kernel cannot run in the CPU emulation tier, so this file restates that integer arithmetic and the host's
shared-memory budget and checks them at the H100's 132 SMs."""
import itertools

import pytest

G = 132
STAGE_BYTES = 16384          # STC_STAGE_BYTES
NS_MIN = 4                   # STC_NS_MIN
TT_PITCH = 132               # STC_TT_PITCH
QL_MAX = 64                  # STC_QL_MAX
SMEM_LIMIT = 227 * 1024 - 3072


def lo(U, G, b):
    return (U * b) // G


def geometry(n, C, fs):
    npx = fs * fs
    kbt, kba, nchk = (npx + 31) // 32, C // 32, C // 128
    return kbt, kba, nchk, nchk * n * kbt


def smax_of(n, C, fs):
    kbt, _, _, UT = geometry(n, C, fs)
    return max(len({(u // kbt) % n for u in range(lo(UT, G, b), lo(UT, G, b + 1))}) for b in range(G))


def nbt_of(n, C, fs):
    kbt, kba, _, UT = geometry(n, C, fs)
    return max(kba, min((UT + G - 1) // G, n * kbt))


CASES = list(itertools.product(range(32, 51), [128, 256, 512], [18, 22]))


@pytest.mark.parametrize("n,C,fs", CASES)
def test_rt_slots_cover_each_range_once(n, C, fs):
    kbt, _, _, UT = geometry(n, C, fs)
    per_chunk = n * kbt
    nbt = nbt_of(n, C, fs)
    for b in range(G):
        t_lo, t_hi = lo(UT, G, b), lo(UT, G, b + 1)
        nslots = min(t_hi - t_lo, per_chunk)
        assert nslots <= nbt
        # build_rt: slot s holds the pair of unit t_lo + s
        built = [((t_lo + s) % per_chunk) // kbt for s in range(nslots)], [((t_lo + s) % per_chunk) % kbt for s in range(nslots)]
        pairs = list(zip(*built))
        assert len(set(pairs)) == nslots                                    # one slot per pair
        # the consumer: running slot counter wrapping at n * KBT; unit u = (chunk, sample, pixel block) must find its own pair
        sl = 0
        for u in range(t_lo, t_hi):
            assert pairs[sl] == ((u % per_chunk) // kbt, u % kbt)
            sl += 1
            if sl == per_chunk:
                sl = 0
        assert {((u % per_chunk) // kbt, u % kbt) for u in range(t_lo, t_hi)} == set(pairs)


@pytest.mark.parametrize("n,C,fs", CASES)
def test_shared_memory_fits_the_wgmma_path(n, C, fs):
    """launch_sd_tc's budget: at least STC_NS_MIN stages next to the B-tile region and the per-sample state."""
    kbt, kba, _, UT = geometry(n, C, fs)
    npos = (fs + 1) ** 2
    smax = smax_of(n, C, fs)
    assert smax <= 16
    slice_max = (C * 4 + G - 1) // G + 1
    fixed = (1024 + nbt_of(n, C, fs) * 4096 + 16 * TT_PITCH * 4 + 2 * slice_max * 16 + smax * 6 * npos * 4 + smax * (QL_MAX + 1) * 4
             + 64)
    assert fixed + NS_MIN * STAGE_BYTES <= SMEM_LIMIT
