"""CPU: the tile plan of the persistent tensor-core conv kernel (t2_plan in csrc/conv_tc2.cu), through the host-only plan
query avc_conv_block_tc_plan.  No kernel runs: the plan is computed for a given SM count.

* a sweep over batch, channels, taps, stride, length and fold: every plan that is not rejected stays inside the limits
  the kernel relies on (a kernel instance exists, the MMAs read only staged rows plus the stage's slack, tensor-map box
  dimensions, shared memory, ring depth, epilogue tile);
* every descriptor the engine sends to avc_conv_block_tc in a training step and in inference gets a plan: the engine
  runs on the CPU against a stand-in for the C ABI that hands each such descriptor to the plan query;
* the case list of tests/test_gpu_tc2_exact.py reaches every kernel instance and plan feature at 132 and 114 SMs.
"""
import ctypes as C
import math

import pytest
import torch

import oracle.ae_oracle as orc
from test_gpu_tc2_exact import FEATURES, INSTANCES, cases, features, geometry, make_desc, plan_of

SMS = (132, 114)
SLACK_ROWS = 32          # rows of 16 bytes every stage keeps past its last plane
BOX_MAX = 256            # elements per tensor-map box dimension
SMEM_OPTIN = 227 * 1024  # H100: dynamic + static shared memory per block
STATIC_SMEM = 4 * 8 * 8  # the kernel's four mbarrier arrays of 8 stages


@pytest.fixture(scope="module")
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


def desc(B, Cin, Cout, K, T, stride=1, fold=False, zero=False, norm=False):
    """A conv block (reflect or zero padding) or, with fold, the folded data gradient of a stride-1 block whose output
    gradient has T steps -- built the way engine.py builds them.  Pointers are stand-ins (the query reads none)."""
    from adaptive_voice_conversion_b200 import _lib as L
    pl, pr = K // 2, K // 2 - (1 if K % 2 == 0 else 0)
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups = B, Cin, Cout, K, stride, 1
    d.in_, d.w_tc, d.out = 1 << 20, 1 << 20, 1 << 20
    d.in_bstride, d.eps = Cin * T, 1e-5
    d.Tin = T
    if fold:
        d.pad_left, d.pad_mode, d.Tout, d.out_T = K - 1, L.PAD_ZERO, T + K - 1, T
        d.flags = L.F_FOLD | (pl << 8) | (pr << 16)
    else:
        d.pad_left, d.pad_mode, d.Tout = pl, L.PAD_ZERO if zero else L.PAD_REFLECT, (T + pl + pr - K) // stride + 1
        d.norm = int(norm)
    return d


def check_plan(d, p):
    """The conditions the kernel relies on, for the plan p of descriptor d."""
    K, S = d.K, d.stride
    assert (p.N, p.N_last if p.nchunk > 1 else p.N) in INSTANCES and p.instance == INSTANCES.index(
        (p.N, p.N_last if p.nchunk > 1 else p.N)), (p.N, p.N_last, p.nchunk)
    ncol = (p.TT - 1) * S + 1                      # accumulator columns one sample's outputs occupy
    assert p.R == ncol + K - 1 and p.srows == p.G * p.R
    cols = (p.nchunk - 1) * p.N + p.N_last           # accumulator columns the chunks compute
    assert cols >= (p.G - 1) * p.R + ncol            # ... cover every output column of every stacked sample
    assert cols - p.N_last < (p.G - 1) * p.R + ncol  # ... and the last chunk is not empty
    # the last chunk's MMAs read rows up to cols + K - 1 of the last plane: staged rows plus the stage's slack
    assert cols + K - 1 <= p.srows + SLACK_ROWS, (cols, K, p.srows)
    assert p.nchunk == 1 or (d.flags & 4 and p.N == 128 and p.G == 1)
    assert 1 <= p.G <= 8 and p.G <= d.B
    # tensor-map boxes: input (4, R, G, 2 hs), weights (256, 2, 2, K) when hs == 1
    assert p.R <= BOX_MAX and 2 * p.hs <= BOX_MAX and p.G <= BOX_MAX
    nhalf = d.Cin // 8
    assert p.hs in (1, 2, 4) and p.hs <= max(nhalf, 1) and p.nst == math.ceil(nhalf / p.hs)
    w_bytes = K * 4096 if p.hs == 1 else (p.hs // 2) * K * 8192
    assert p.stage_bytes >= w_bytes + 2 * p.hs * p.srows * 16 + SLACK_ROWS * 16 and p.stage_bytes % 1024 == 0
    assert p.smem_bytes <= p.smem_max and p.smem_max + STATIC_SMEM <= SMEM_OPTIN
    assert p.smem_bytes >= p.nstage * p.stage_bytes + 32 * p.P * 16
    assert 2 <= p.nstage <= 8
    # epilogue tile: G samples x Ts columns per 4-channel chunk, pitch == 1 mod 8
    assert p.Ts == p.TT and p.P >= p.G * p.Ts and p.P % 8 == 1
    # time tiles cover the output exactly; only blocks without whole-sample statistics are time-tiled
    assert (p.ntt - 1) * p.TT < d.Tout <= p.ntt * p.TT
    assert p.ntt == 1 or (not d.norm and not d.shuffle and not (d.flags & 4) and p.G == 1)
    assert p.mtiles == math.ceil(d.Cout / 128) and p.ntiles == math.ceil(d.B / p.G) * p.ntt * p.mtiles


def run(lib, d, sms):
    from adaptive_voice_conversion_b200 import _lib as L
    rc, p = plan_of(lib, d, sms)
    if rc != 0:
        assert rc == L.ERR_UNSUPPORTED, (rc, L.last_error())
        assert L.last_error().startswith("avc_conv_block_tc"), L.last_error()
        assert "no kernel instance" not in L.last_error(), L.last_error()   # a plan without a kernel is a planner bug
        return None
    check_plan(d, p)
    return p


BS = (1, 2, 3, 7, 8, 9, 131, 132, 133, 256, 1056)
CINS = (16, 32, 80, 128, 256, 1104)
COUTS = (80, 128, 256, 1104)
T_EDGES = (1, 2, 5, 16, 17, 64, 65, 127, 128, 129, 141, 143, 144, 145, 160, 200, 248, 249, 250, 256, 257, 288, 300, 512, 600)


@pytest.mark.parametrize("sms", SMS)
def test_plan_sweep(lib, sms):
    """Every combination at the edge lengths, and every length 1..600 with the other sizes cycling."""
    n = ok = 0
    shapes = [(B, Cin, Cout) for B in BS for Cin in CINS for Cout in COUTS]
    for K in range(1, 9):
        for stride, fold in ((1, False), (2, False), (1, True)):
            for T in T_EDGES:
                for B, Cin, Cout in shapes:
                    p = run(lib, desc(B, Cin, Cout, K, T, stride, fold, zero=(B % 2 == 0), norm=(Cin == 128)), sms)
                    n, ok = n + 1, ok + (p is not None)
            for T in range(1, 601):
                B, Cin, Cout = shapes[(T * 7 + K * 31 + stride) % len(shapes)]
                p = run(lib, desc(B, Cin, Cout, K, T, stride, fold, zero=(T % 2 == 1)), sms)
                n, ok = n + 1, ok + (p is not None)
    assert ok > n // 2, (ok, n)


def test_plan_rejects_what_the_kernel_cannot_tile(lib):
    from adaptive_voice_conversion_b200 import _lib as L
    assert run(lib, desc(2, 128, 128, 5, 200, norm=True), 132) is None      # InstanceNorm over a time-tiled sample
    assert "time tiles" in L.last_error()
    assert run(lib, desc(2, 128, 128, 5, 253, fold=True), 132) is None      # folded sample of 257 staged rows
    assert run(lib, desc(2, 128, 128, 5, 2), 132) is None                   # reflect padding 2 of 2 steps
    assert "reflect padding" in L.last_error()
    d = desc(2, 128, 128, 5, 64)
    d.in_ = (1 << 20) + 4                                                    # tensor-map operand not 16-byte aligned
    assert run(lib, d, 132) is None
    d = desc(2, 120, 128, 5, 64)                                             # argument check of the launch: Cin % 16
    assert run(lib, d, 132) is None and "Cin % 16" in L.last_error()


def test_plan_depends_on_the_sm_count(lib):
    """Samples per tile follow the SM count: 8 x 132 samples of 16 steps fill 132 CTAs with one round of G = 8 tiles;
    on 114 SMs that would take two rounds, and the planner takes two rounds of narrower tiles instead."""
    d = desc(8 * 132, 16, 128, 5, 16)
    p132, p114 = run(lib, d, 132), run(lib, d, 114)
    assert (p132.G, p132.N, p132.ntiles) == (8, 160, 132)
    assert p114.G < 8 and 114 < p114.ntiles <= 2 * 114


# ------------------------------------------------------------------ what the engine sends
class PlanLib:
    """Stand-in for the C ABI: every call succeeds; avc_conv_block_tc hands its descriptor to the real plan query and
    records the rejections."""

    def __init__(self, real, sms):
        self.real, self.sms = real, sms
        self.n, self.rejected, self.instances = 0, [], set()

    def avc_conv_block_tc(self, dref, status, stream):
        from adaptive_voice_conversion_b200 import _lib as L
        d = dref._obj
        rc, p = plan_of(self.real, d, self.sms)
        self.n += 1
        if rc != 0:
            self.rejected.append((d.B, d.Cin, d.Cout, d.K, d.stride, d.Tin, d.Tout, int(d.flags), L.last_error()))
        else:
            check_plan(d, p)
            self.instances.add((p.N, p.N_last if p.nchunk > 1 else p.N))
        return 0

    def __getattr__(self, name):
        def f(*a):
            if name in ("avc_tc_packed_floats", "avc_wgrad_tc_scratch_floats", "avc_conv_wgrad_scratch_floats"):
                return 64
            if name == "avc_wgrad_acc_floats":
                return a[2] * a[1] * (((a[0] + 127) // 128) * 128)
            return 0
        return f


def cpu_engine(monkeypatch, lib, sms, c_in=80, cfg=None, precision="tf32", stand_in=PlanLib):
    from adaptive_voice_conversion_b200 import engine as E
    cfg = orc.default_config(c_in) if cfg is None else cfg
    e = object.__new__(E.Engine)      # the real constructor insists on a CUDA device
    e.cfg, e.dev, e.lib, e.packed, e.debug = cfg, torch.device("cpu"), stand_in(lib, sms), {}, None
    e.precision, e.tc_status, e._packed_key = precision, torch.zeros(1, dtype=torch.int32), None
    e._init_options()
    monkeypatch.setattr(E.Engine, "stream", property(lambda self: 0))
    monkeypatch.setattr(E.Engine, "zeros", lambda self, *shape: torch.zeros(shape))
    P = orc.init_state(cfg, seed=0)
    e.pack_weights(P, need_dgrad=True)
    return e, P


def train_step(e, P, B, T):
    from adaptive_voice_conversion_b200.engine import A4
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    x = torch.empty(B, e.cfg["SpeakerEncoder"]["c_in"], T)
    emb, cs = e.speaker_fwd(P, x, True)
    mu4, ls4, ce = e.content_fwd(P, x, True)
    eps = torch.empty(B, mu4.C, mu4.T)
    mu, ls, z4 = e.reparam_fwd(mu4, ls4, eps)
    dec4, cd = e.decoder_fwd(P, z4, emb, True)
    dz4, demb = e.decoder_bwd(P, G, cd, A4.empty(dec4.B, dec4.C, dec4.T, e.dev))
    dmu4, dls4 = e.reparam_bwd(dz4, ls4, eps, torch.zeros_like(mu), torch.zeros_like(ls))
    e.content_bwd(P, G, ce, dmu4, dls4)
    e.speaker_bwd(P, G, cs, demb)


@pytest.mark.parametrize("sms", SMS)
def test_engine_training_descriptors_all_plan(monkeypatch, lib, sms):
    """Forward blocks, stride-2 parity data gradients and folded / plain data gradients of a training step, for the
    default segment (128 frames) and segment_size 64, 200 and 232, at B = 1, 16 and 256, with the fused fold on and off;
    also the 512-mel config.  (Training lengths are the ones the decoder reproduces: multiples of 8.)"""
    seen = set()
    for c_in, segs in ((80, (64, 128, 200, 232)), (512, (128,))):
        e, P = cpu_engine(monkeypatch, lib, sms, c_in)
        for fold in (True, False):
            e.fold_fused = fold
            for T in segs:
                for B in (1, 16, 256):
                    train_step(e, P, B, T)
        assert e.lib.n > 0 and not e.lib.rejected, e.lib.rejected[:5]
        seen |= e.lib.instances
    # the chunked folded widths are in real use (segment_size 200 / 232)
    assert any(nl != n for n, nl in seen), sorted(seen)


def test_engine_inference_descriptors_all_plan(monkeypatch, lib):
    """One utterance (B = 1) of every length 1..600 frames.  Below 17 frames a reflect padding of the encoders meets a
    sequence shorter than itself -- the reference's F.pad(mode="reflect") fails there too -- and only that is rejected."""
    e, P = cpu_engine(monkeypatch, lib, 132)
    for T in range(1, 601):
        e.lib.rejected.clear()
        x = torch.empty(1, 80, T)
        with torch.no_grad():
            emb, _ = e.speaker_fwd(P, x, False)
            mu4, ls4, _ = e.content_fwd(P, x, False)
            e.decoder_fwd(P, mu4, emb, False)
        if T >= 17:
            assert not e.lib.rejected, (T, e.lib.rejected[:3])
        else:
            assert all("reflect padding" in r[-1] for r in e.lib.rejected), (T, e.lib.rejected[:3])
    assert {(96, 96), (112, 112)} <= e.lib.instances


@pytest.mark.parametrize("sms", SMS)
def test_gpu_case_list_covers_every_instance_and_feature(lib, sms):
    fake = {k: 1 << 20 for k in ("x", "out", "c", "stats", "bias", "cond", "res", "mask", "w", "w_even", "w_odd")}
    covered = set()
    for case in cases(sms):
        for g, par in geometry(case):
            d = make_desc(case, g, par, fake)
            p = run(lib, d, sms)
            assert p is not None, case.id
            covered |= features(case, g, par, p, sms)
    assert [f for f in FEATURES if f not in covered] == []
    assert {f for f in covered if f[0] == "instance"} == {("instance", n, nl) for n, nl in INSTANCES}
