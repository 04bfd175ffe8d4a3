"""GPU: edge cases of the weight-gradient kernel's window staging, against the float64 reference of
test_gpu_wgrad_exact.py at its tolerance.

conv_wgrad_wgmma_kernel stages x one (4-channel chunk, 4-row plane) window per thread; a staging warpgroup is two halves
that stage different chunks (4 halves at K <= 6, 2 at K = 7, 8), and where two register sets fit a half loads its next
chunk before it stores the current one.  The cases below reach what that mapping adds and the exact-operand sweep does
not: slices of one to three chunks (fewer chunks than halves, halves with no chunk or with a prefetch that has nothing
to load), a last chunk that ends half-way (its planes 4..7 past the slice's rows), Tout = 8 at K = 7 and 8 (every
window of a sample reflects at its left or its right edge, with and without the prefetch), and stride 2 at Tout = 64
with the prefetch (K <= 4) and without it (K = 6).  test_window_cases_reach_the_edges checks those claims against the
plan mirror.
"""
import pytest
import torch

from test_gpu_wgrad_exact import TOL, Case, cdiv, data, errors, eng, guarded, guards_intact, launch, tc_plan  # noqa: F401

pytestmark = pytest.mark.gpu

WG_ROWS = 32


def halves(K):
    return 4 if K <= 6 else 2


CASES = [
    Case("tc", 1, 128, 128, 5, 32),           # one chunk per slice
    Case("tc", 2, 64, 128, 7, 32),            # two chunks, K = 7: two halves, prefetch with nothing left to load
    Case("tc", 3, 128, 128, 3, 32),           # three chunks: one half idle
    Case("tc", 1, 80, 128, 2, 16),            # one chunk, half past the slice's rows
    Case("tc", 5, 128, 128, 4, 16),           # G = 8 > B: 80 rows, the last of 3 chunks ends half-way
    Case("tc", 4, 128, 128, 8, 8),            # Tout = 8, K = 8: reflect at both edges of every sample
    Case("tc", 9, 80, 128, 7, 8, strided=True),   # Tout = 8, K = 7 with the prefetch
    Case("tc", 6, 128, 128, 4, 128, stride=2),    # stride 2, Tout = 64, prefetch
    Case("tc", 3, 128, 128, 6, 128, stride=2),    # stride 2, Tout = 64, no prefetch
]


def chunks_per_slice(case):
    G, ns, _ = tc_plan(case.B, case.Cin, case.Cout, case.K, case.Tout, case.stride)
    per = cdiv(cdiv(case.B, G), ns) * G
    return [cdiv(min(per, case.B - s * per) * case.Tout, WG_ROWS) for s in range(ns)]


def test_window_cases_reach_the_edges():
    reach = set()
    for c in CASES:
        for n in chunks_per_slice(c):
            if n < halves(c.K):
                reach.add(("fewer chunks than halves", n))
        G, ns, _ = tc_plan(c.B, c.Cin, c.Cout, c.K, c.Tout, c.stride)
        per = cdiv(cdiv(c.B, G), ns) * G
        if any((min(per, c.B - s * per) * c.Tout) % WG_ROWS == 16 for s in range(ns)):
            reach.add("last chunk ends half-way")
        if c.Tout == 8 and c.K in (7, 8):
            reach.add(("Tout 8 reflect", c.K))
        if c.stride == 2 and c.Tout == 64:
            reach.add(("stride 2 Tout 64", c.K <= 4))
    want = {("fewer chunks than halves", n) for n in (1, 2, 3)} | {"last chunk ends half-way"}
    want |= {("Tout 8 reflect", 7), ("Tout 8 reflect", 8), ("stride 2 Tout 64", True), ("stride 2 Tout 64", False)}
    assert want <= reach, want - reach


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_wgrad_window_edges(eng, case):  # noqa: F811
    x, dc, ref, aref, pre = data(case)
    dbuf, dw = guarded(pre.numel())
    dw.copy_(pre.flatten())
    sbuf = launch(eng, case, x, dc, dw)
    torch.cuda.synchronize()
    assert guards_intact(dbuf), "write outside dw"
    assert guards_intact(sbuf), "write outside the scratch region"
    eb, er = errors(dw.view_as(pre), pre, ref, aref)
    assert eb < TOL["tc"], f"max error {eb:.3e} of sum |dc||x| (relative to max |ref|: {er:.3e}; tolerance {TOL['tc']:.0e})"
