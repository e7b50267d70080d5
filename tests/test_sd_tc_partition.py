"""Invariants of the unit decomposition of the tensor-core (wgmma) steepest-descent kernel (pytracking_b200/csrc/sd_tc.cu).

The kernel deals the 128 x 32 operand tiles ("units") of a sweep to the CTAs as contiguous ranges [lo(b), lo(b+1)) with
lo(b) = floor(b U / G), and every consumer re-derives, with integer arithmetic only, which CTA produced which partial:
owner(u), the segment starts inside a (sample, pixel tile) run, the contributors of a gradient chunk.  This file restates that
arithmetic (part_lo / part_owner in the kernel) and checks the properties the kernel's fixed-order reductions rely on."""
import itertools

import pytest


def lo(U, G, b):
    return (U * b) // G


def owner(U, G, u):
    return ((u + 1) * G - 1) // U


CASES = [(U, G) for U, G in itertools.product([1, 7, 22, 148, 149, 660, 1100, 2200, 2400, 3200, 9600, 12345], [1, 4, 132, 148, 160])]


@pytest.mark.parametrize("U,G", CASES)
def test_ranges_partition_the_units(U, G):
    seen = []
    for b in range(G):
        seen.extend(range(lo(U, G, b), lo(U, G, b + 1)))
    assert seen == list(range(U))                                   # every unit exactly once, in order
    assert max(lo(U, G, b + 1) - lo(U, G, b) for b in range(G)) - min(lo(U, G, b + 1) - lo(U, G, b) for b in range(G)) <= 1


@pytest.mark.parametrize("U,G", CASES)
def test_owner_is_the_cta_whose_range_holds_the_unit(U, G):
    for u in range(U):
        b = owner(U, G, u)
        assert 0 <= b < G and lo(U, G, b) <= u < lo(U, G, b + 1)


@pytest.mark.parametrize("G", [132, 114, 148], ids=["h100_sxm", "h100_pcie", "g148"])
@pytest.mark.parametrize("n,C,fs", [(1, 512, 18), (3, 256, 18), (15, 512, 18), (50, 512, 18), (50, 128, 22), (15, 512, 22), (33, 384, 18)])
def test_apply_segments_and_gradient_contributors(n, C, fs, G):
    npx = fs * fs
    kbt, npt, kba, nchk = (npx + 31) // 32, (npx + 127) // 128, C // 32, C // 128
    UA, UT = n * npt * kba, nchk * n * kbt
    # apply sweep: a segment starts at channel block 0 of a (sample, pixel tile) run and at every range boundary inside it;
    # the consumer's test "lo(owner(u)) == u" must find exactly the segments the producers write
    written = set()
    for b in range(G):
        a, e = lo(UA, G, b), lo(UA, G, b + 1)
        for u in range(a, e):
            if u == a or u % kba == 0:
                written.add(u)
    derived = {u for u in range(UA) if u % kba == 0 or lo(UA, G, owner(UA, G, u)) == u}
    assert derived == written
    assert max(sum(1 for u in range(r * kba, (r + 1) * kba) if u in written) for r in range(n * npt)) <= kba
    # adjoint sweep: the contributors of chunk c are the non-empty ranges between the owners of its first and last unit,
    # and a range never spans more chunks than the kernel has accumulators for (STC_MAXCH = 4)
    per_chunk = n * kbt
    for c in range(nchk):
        bf, bl = owner(UT, G, c * per_chunk), owner(UT, G, (c + 1) * per_chunk - 1)
        contributors = [b for b in range(bf, bl + 1) if lo(UT, G, b + 1) > lo(UT, G, b)]
        touching = [b for b in range(G) if lo(UT, G, b + 1) > lo(UT, G, b) and
                    lo(UT, G, b) < (c + 1) * per_chunk and lo(UT, G, b + 1) > c * per_chunk]
        assert contributors == touching
        for b in contributors:
            assert 0 <= c - lo(UT, G, b) // per_chunk < 4
    # state slots: the distinct samples an adjoint range touches (the host sizes shared memory for the maximum, at most 16)
    smax = 0
    for b in range(G):
        a, e = lo(UT, G, b), lo(UT, G, b + 1)
        smax = max(smax, len({(u // kbt) % n for u in range(a, e)}))
    assert 1 <= smax <= 16
    # every sample has exactly one owner CTA (the one holding unit (chunk 0, sample, block 0))
    assert sorted(owner(UT, G, s * kbt) for s in range(n)) == [owner(UT, G, s * kbt) for s in range(n)]
