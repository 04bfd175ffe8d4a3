"""CPU: which weight-gradient kernel the engine picks for each conv of a training step, and whether the GPU case list of
tests/test_gpu_wgrad_exact.py stands for those launches.  No kernel runs: the engine runs against the stand-in C ABI of
tests/test_conv_tc2_plan.py, whose size queries here are the library's real, host-only ones.
"""
import ctypes as C

import pytest

from test_conv_tc2_plan import PlanLib, cpu_engine, train_step
from test_gpu_wgrad_exact import CASES, case_keys, desc_keys, make_desc, simt_plan, tc_plan, tc_supported


@pytest.fixture(scope="module")
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


class WgradLib(PlanLib):
    """Records every weight-gradient launch with the kernel that serves it."""

    def __init__(self, real, sms):
        super().__init__(real, sms)
        self.launches = []

    def _record(self, kernel, dref):
        d = dref._obj
        self.launches.append((kernel, d.B, d.Cin, d.Cout, d.K, d.Tin, d.Tout, d.stride,
                              d.x_bstride != d.Cin * d.Tin or d.dc_bstride != d.Cout * d.Tout))
        return 0

    def avc_wgrad_tc_scratch_floats(self, dref):
        return self.real.avc_wgrad_tc_scratch_floats(dref)

    def avc_conv_wgrad_scratch_floats(self, dref):
        return self.real.avc_conv_wgrad_scratch_floats(dref)

    def avc_conv_wgrad_tc(self, dref, scratch, status, stream):
        return self._record("tc", dref)

    def avc_conv_wgrad(self, dref, scratch, stream):
        return self._record("simt", dref)


def engine_launches(monkeypatch, lib, c_in, segs, batches=(1, 16, 256)):
    e, P = cpu_engine(monkeypatch, lib, 132, c_in)
    e.lib = WgradLib(lib, 132)
    out = {}
    for T in segs:
        for B in batches:
            e.lib.launches.clear()
            train_step(e, P, B, T)
            out[(T, B)] = list(e.lib.launches)
    return out


def test_default_segment_runs_every_weight_gradient_on_the_tensor_cores(monkeypatch, lib):
    """At the default segment (128 frames) every weight gradient of a step is served by avc_conv_wgrad_tc, the kernel
    with the fixed-order reduction -- for 80 and 512 mels."""
    for c_in in (80, 512):
        for (T, B), launches in engine_launches(monkeypatch, lib, c_in, (128,)).items():
            assert len(launches) == 58, (c_in, T, B, len(launches))
            assert all(l[0] == "tc" for l in launches), (c_in, B, [l for l in launches if l[0] != "tc"])


def test_engine_launches_are_covered_by_the_gpu_cases(monkeypatch, lib):
    """Every feature key of every weight-gradient launch of a training step (80 mels at segments 64/128/200/244 and 512
    mels at 128, B = 1/16/256) is reached by a case of the GPU list; longer segments do reach the FFMA kernel."""
    covered = set().union(*(case_keys(c) for c in CASES))
    kernels, missing = set(), {}
    for c_in, segs in ((80, (64, 128, 200, 244)), (512, (128,))):
        for (T, B), launches in engine_launches(monkeypatch, lib, c_in, segs).items():
            for kernel, B_, Cin, Cout, K, Tin, Tout, stride, strided in launches:
                kernels.add(kernel)
                assert (kernel == "tc") == tc_supported(B_, Cin, Cout, K, Tin, Tout, stride)
                for k in desc_keys(kernel, B_, Cin, Cout, K, Tin, Tout, stride, strided) - covered:
                    missing.setdefault(k, (c_in, T, B, Cin, Cout, K, Tout, stride))
    assert kernels == {"tc", "simt"}
    assert not missing, missing


def test_plan_mirrors_match_the_library(lib):
    """tc_plan / simt_plan (the test module's copies of the launch plans) give the library's scratch sizes, for the GPU
    cases and a sweep of shapes; the tensor-core size query refuses exactly the shapes tc_supported refuses."""
    from test_gpu_wgrad_exact import Case
    shapes = list(CASES)
    for B in (1, 2, 5, 17, 64, 256, 1000):
        for Cin, Cout in ((16, 128), (80, 128), (128, 80), (128, 256), (512, 128), (1104, 128), (1536, 512)):
            for K in (1, 2, 5, 8):
                for Tin, stride in ((8, 1), (24, 1), (37, 1), (64, 1), (128, 1), (200, 1), (15, 2), (64, 2), (129, 2), (300, 2)):
                    shapes.append(Case("tc", B, Cin, Cout, K, Tin, stride))
    for c in shapes:
        d = make_desc(c, 1 << 20, 1 << 20, 1 << 20)
        n_tc = int(lib.avc_wgrad_tc_scratch_floats(C.byref(d)))
        if tc_supported(c.B, c.Cin, c.Cout, c.K, c.Tin, c.Tout, c.stride):
            G, ns, coutp = tc_plan(c.B, c.Cin, c.Cout, c.K, c.Tout, c.stride)
            assert n_tc == ns * c.K * c.Cin * coutp, c.id
        else:
            assert n_tc == -1, c.id
        ns, coutp = simt_plan(c.B, c.Cin, c.Cout, c.K, c.Tout)
        assert int(lib.avc_conv_wgrad_scratch_floats(C.byref(d))) == ns * c.K * c.Cin * coutp, c.id
    for c in CASES:
        assert (c.kernel == "tc") == tc_supported(c.B, c.Cin, c.Cout, c.K, c.Tin, c.Tout, c.stride), c.id
