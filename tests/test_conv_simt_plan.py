"""CPU: the tile plan of the exact-fp32 FFMA conv-block kernel (simt_plan in csrc/conv_simt.cu), through the host-only
plan query avc_conv_block_fwd_plan.  No kernel runs.

* a sweep over batch, channels, taps, stride, zero insertion, length, InstanceNorm and pixel shuffle: every plan that is
  not rejected stays inside the limits the kernel relies on (a kernel instance exists, segments tile the CTA, the staged
  input rows hold every thread's read window, the grid covers batch and channels, shared memory);
* every descriptor the engine sends to avc_conv_block_fwd at precision "fp32" -- a training step, and inference of one
  utterance -- gets a plan and carries nothing the query refuses, and the plan features those launches reach are a subset
  of what the case list of tests/test_gpu_conv_simt_exact.py reaches;
* that case list reaches every kernel instance and every entry of its FEATURES.
"""
import ctypes as C

import pytest
import torch

from test_conv_tc2_plan import PlanLib, cpu_engine, train_step
from test_gpu_conv_simt_exact import CASES, FEATURES, launch_keys, make_desc, plan_of, rejected_descs

SMEM_STATIC_MAX = 48 * 1024   # the kernel's dynamic shared memory stays within the default limit
CK = 8                        # input channels per shared-memory stage
FAKE = {k: 1 << 20 for k in ("x", "w", "out", "c", "stats", "bias", "cond", "res", "mask")}


@pytest.fixture(scope="module")
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


def cdiv(a, b):
    return -(-a // b)


def check_plan(d, p):
    """The conditions the kernel relies on, for the plan p of descriptor d."""
    from adaptive_voice_conversion_b200 import _lib as L
    K, S = d.K, d.stride
    assert 0 <= p.instance < len(L.SIMT_INSTANCES) and L.SIMT_INSTANCES[p.instance] == (K, S, p.TCO, p.TT), (p.instance, K, S, p.TT)
    assert p.TCO * p.TT == 256 * 64                                # 256 threads of 8 x 8 outputs
    assert p.seg_out * p.nseg == p.TT and p.seg_out >= 8 and p.seg_out & (p.seg_out - 1) == 0
    if p.tiled:
        assert not d.norm and p.nseg == 1 and p.TT == 128
        assert (p.ntt - 1) * p.TT < d.Tout <= p.ntt * p.TT
        assert p.grid_x == d.B * p.ntt
    else:
        assert p.ntt == 1 and p.seg_out >= d.Tout                 # a whole sample in one segment
        assert p.seg_out // 2 < max(d.Tout, 8) or p.TT == 256      # ... of the narrowest power of two
        assert p.grid_x == cdiv(d.B, p.nseg)
    assert (p.grid_y - 1) * p.TCO < d.Cout <= p.grid_y * p.TCO
    # InstanceNorm statistics: a shuffle reduction over the seg_out / 8 lanes of a segment, inside one row of threads
    nlanes, ntx = p.seg_out // 8, p.TT // 8
    assert nlanes <= 32 and ntx % nlanes == 0 and (ntx % 32 == 0 or 32 % ntx == 0)
    # staging: nseg segments of segp floats; one segment holds the input window of seg_out outputs
    assert p.segp == cdiv(p.seg_out * S + K - 1, 4) * 4 and p.nseg * p.segp <= p.xrow
    # every thread reads 4 * ceil((7 S + K) / 4) floats from tl * S of its segment (tl = 8 * lane in the segment)
    nx4 = cdiv(7 * S + K, 4)
    assert (p.nseg - 1) * p.segp + (p.seg_out - 8) * S + 4 * nx4 <= p.xrow
    assert p.smem_bytes == 4 * CK * (p.xrow + K * p.TCO) and p.smem_bytes <= SMEM_STATIC_MAX


def run(lib, d):
    from adaptive_voice_conversion_b200 import _lib as L
    rc, p = plan_of(lib, d)
    if rc != 0:
        assert rc == L.ERR_UNSUPPORTED, (rc, L.last_error())
        assert L.last_error().startswith("avc_conv_block_fwd:"), L.last_error()
        assert "no kernel" not in L.last_error(), L.last_error()     # a plan without a kernel is a planner bug
        return None
    check_plan(d, p)
    return p


def desc(B, Cin, Cout, K, T, stride=1, ups=1, norm=False, shuffle=False):
    """A forward block (ups 1, reflect padding) or a data gradient (ups = the forward stride, zero padding K - 1) over a
    logical input of T steps (stored T // ups).  Pointers are stand-ins (the query reads none)."""
    from adaptive_voice_conversion_b200 import _lib as L
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups = B, Cin, Cout, K, stride, ups
    d.in_, d.w_packed, d.out, d.w_ld, d.eps = 1 << 20, 1 << 20, 1 << 20, Cout, 1e-5
    pl, pr = K // 2, K // 2 - (1 if K % 2 == 0 else 0)
    if ups == 1:
        d.pad_left, d.pad_mode, d.Tin, d.Tout = pl, L.PAD_REFLECT, T, (T + pl + pr - K) // stride + 1
        d.norm, d.shuffle = int(norm), int(shuffle)
    else:
        d.pad_left, d.pad_mode, d.Tin, d.Tout = K - 1, L.PAD_ZERO, max(T // ups, 1), T + K - 1
    d.in_bstride = Cin * d.Tin
    return d


BS = (1, 2, 3, 7, 16, 17, 33, 256)
CHANNELS = ((4, 8), (36, 128), (80, 128), (84, 96), (128, 80), (128, 256), (1104, 128), (128, 1024))
T_EDGES = (1, 2, 3, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 127, 128, 129, 130, 200, 255, 256, 257, 258,
           300, 511, 512, 513, 1000)


def test_plan_sweep(lib):
    """Every edge length at every K, stride / zero insertion, norm and shuffle, the batch and channels cycling."""
    n = ok = 0
    shapes = [(B, ci, co) for B in BS for ci, co in CHANNELS]
    for K in range(1, 9):
        for stride, ups in ((1, 1), (2, 1), (1, 2)):
            for T in T_EDGES:
                for norm, shuffle in ((False, False), (True, False), (True, True), (False, True)):
                    B, Cin, Cout = shapes[(T * 7 + K * 31 + stride + 3 * norm + 5 * shuffle) % len(shapes)]
                    if shuffle and (ups != 1 or Cout % 8):
                        continue
                    p = run(lib, desc(B, Cin, Cout, K, T, stride, ups, norm and ups == 1, shuffle))
                    n, ok = n + 1, ok + (p is not None)
    assert ok > n // 2, (ok, n)
    # every instance at every batch and channel shape
    for B, Cin, Cout in shapes:
        for K, S, T, norm in ((1, 1, 200, True), (5, 1, 150, True), (5, 2, 400, True), (3, 1, 700, False), (5, 2, 9, False)):
            assert run(lib, desc(B, Cin, Cout, K, T, S, 1, norm)) is not None


def test_plan_rejects_what_the_kernel_cannot_run(lib):
    from adaptive_voice_conversion_b200 import _lib as L
    for what, d in rejected_descs(FAKE):
        rc, _ = plan_of(lib, d)
        assert rc == L.ERR_UNSUPPORTED and L.last_error().startswith("avc_conv_block_fwd:"), (what, rc, L.last_error())
    assert run(lib, desc(2, 128, 128, 5, 300, norm=True)) is None and "Tout 300" in L.last_error()
    assert run(lib, desc(2, 128, 128, 3, 200, norm=True)) is None and "K 3" in L.last_error()
    assert run(lib, desc(2, 128, 128, 3, 200, stride=2)) is None                 # stride 2 only at K = 5
    d = desc(2, 128, 128, 5, 64)
    d.flags = L.F_IN_TF32                                                         # a hint, accepted
    assert run(lib, d) is not None
    d.w_ld = 124                                                                  # w_ld < Cout
    assert plan_of(lib, d)[0] == L.ERR_INVALID
    d = desc(2, 128, 128, 5, 64)
    d.w_packed = None
    assert plan_of(lib, d)[0] == L.ERR_INVALID and "null" in L.last_error()


# ------------------------------------------------------------------ what the engine sends
class SimtLib(PlanLib):
    """Stand-in C ABI that hands every avc_conv_block_fwd descriptor to the real plan query and records its features."""

    def __init__(self, real):
        super().__init__(real, 132)
        self.n_fwd, self.keys = 0, set()

    def avc_conv_block_fwd(self, dref, stream):
        from adaptive_voice_conversion_b200 import _lib as L
        d = dref._obj
        rc, p = plan_of(self.real, d)
        self.n_fwd += 1
        if rc != 0:
            self.rejected.append((d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups, d.Tin, d.Tout, int(d.flags), L.last_error()))
        else:
            check_plan(d, p)
            self.keys |= launch_keys(d, p)
        return 0


def engine_keys(monkeypatch, lib):
    keys = set()
    for c_in in (80, 512):
        e, P = cpu_engine(monkeypatch, lib, 132, c_in)
        e.lib = SimtLib(lib)
        e.precision = "fp32"
        e.packed.clear()
        e.pack_weights(P, need_dgrad=True)
        for B in (1, 16):
            train_step(e, P, B, 128)
        for T in (16, 40, 128, 200, 300, 1000):
            x = torch.empty(1, c_in, T)
            with torch.no_grad():
                emb, _ = e.speaker_fwd(P, x, False)
                mu4, _, _ = e.content_fwd(P, x, False)
                e.decoder_fwd(P, mu4, emb, False)
        assert e.lib.n == 0, "a tensor-core launch at precision fp32"
        assert e.lib.n_fwd > 0 and not e.lib.rejected, e.lib.rejected[:5]
        keys |= e.lib.keys
    return keys


def case_keys(lib):
    keys = set()
    for case in CASES:
        d = make_desc(case, FAKE)
        p = run(lib, d)
        assert p is not None, case.id
        keys |= launch_keys(d, p)
    return keys


def test_engine_fp32_launches_all_plan_and_are_covered_by_the_gpu_cases(monkeypatch, lib):
    """A training step (B = 1 and 16, 128 frames) and one utterance of 16, 40, 128, 200, 300 and 1000 frames, for 80 and 512
    mels: every FFMA launch plans, and what it reaches is reached by the GPU case list."""
    eng = engine_keys(monkeypatch, lib)
    assert {k for k in eng if isinstance(k, tuple) and k[0] == "instance" and len(k) == 2} == {("instance", i) for i in range(12)}
    missing = sorted(eng - case_keys(lib), key=str)
    assert not missing, missing


def test_gpu_case_list_covers_every_instance_and_feature(lib):
    covered = case_keys(lib)
    assert [f for f in FEATURES if f not in covered] == []
