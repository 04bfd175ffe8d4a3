"""CPU: the kernels a training step runs for each conv layer, by precision and segment length, and the segment
lengths the model accepts.

The engine runs a training step on the CPU (test_conv_tc2_plan.cpu_engine, no kernel runs) against a stand-in for the
C ABI that records every launch together with the layer and pass that made it.  Each layer's launches name its routes:

  fwd     tc          fused tensor-core block (avc_conv_block_tc)
          tc_split    plain tensor-core conv, then avc_norm_apply_fwd (statistics and save_c)
          ffma        fused FFMA block (avc_conv_block_fwd)
          ffma_split  plain FFMA conv, then avc_norm_apply_fwd
  normbwd cached      avc_norm_bwd's cached kernel (no pixel shuffle, Tout <= 128: csrc/norm.cu decides)
          plain       its plain kernel; plain_shuffle the pixel-shuffle one
          fused       in the downstream data-gradient conv's epilogue (AVC_F_NORMBWD)
  wgrad   tc, tc_acc  avc_conv_wgrad_tc(_acc) -- when avc_wgrad_tc_scratch_floats (a host query) accepts the shape
          ffma        avc_conv_wgrad
  dgrad   tc_fold     tensor-core transposed conv, halo and residual folded in its epilogue
          tc_s2       the stride-2 parity pair on the tensor cores, then avc_fold_add_fwd
          tc+fold, tc_direct, ffma+fold, ffma_direct: the conv, then avc_fold_add_fwd or nothing (a 1-tap conv)

tests/test_gpu_step_layers.py checks every layer of a step against a float64 restatement; here its case list is shown
to reach every route a step of any length from 64 to 512 frames takes, which its 128-frame cases alone do not.
"""
import types

import pytest

import oracle.ae_oracle as orc
from _sn_ref import sn_config
from test_conv_tc2_plan import PlanLib, cpu_engine, train_step
from test_gpu_step_layers import TRAIN_CASES

SWEEP = range(64, 513, 8)


class RouteLib(PlanLib):
    """PlanLib (every avc_conv_block_tc descriptor must get a tile plan) that also records each avc_* launch with the
    current tag; the weight-gradient shape query is answered by the real library."""

    def __init__(self, real, sms):
        super().__init__(real, sms)
        self.cur, self.calls = None, []

    def avc_conv_block_tc(self, dref, status, stream):
        d = dref._obj
        self.calls.append(("avc_conv_block_tc", self.cur, int(d.flags), int(d.out_tstride)))
        return super().avc_conv_block_tc(dref, status, stream)

    def avc_norm_bwd(self, dref, stream):
        d = dref._obj
        self.calls.append(("avc_norm_bwd", self.cur, bool(d.shuffle), int(d.Tout)))
        return 0

    def avc_wgrad_tc_scratch_floats(self, dref):
        return self.real.avc_wgrad_tc_scratch_floats(dref)

    def __getattr__(self, name):
        f = super().__getattr__(name)
        if not name.startswith("avc_") or name.endswith("_floats"):
            return f

        def call(*a):
            self.calls.append((name, self.cur, None, None))
            return f(*a)
        return call


def _tagging(monkeypatch):
    """Tag every launch with (layer, "fwd" | "bwd" | "wgrad"); a data-gradient conv that ran the upstream block's norm
    backward (fuse_up) is recorded for that block as ("normbwd", "fused")."""
    from adaptive_voice_conversion_b200 import engine as E
    Eng = E.Engine
    conv0, bwd0, wg0 = Eng.conv, Eng.conv_bwd, Eng._wgrad_launch

    def tagged(self, tag, fn):
        prev, self.lib.cur = self.lib.cur, tag
        try:
            return fn()
        finally:
            self.lib.cur = prev

    def conv(self, P, name, xin, **kw):
        return tagged(self, (name, "fwd"), lambda: conv0(self, P, name, xin, **kw))

    def conv_bwd(self, P, G, rec, dy, **kw):
        r = tagged(self, (rec["name"], "bwd"), lambda: bwd0(self, P, G, rec, dy, **kw))
        up = kw.get("fuse_up")
        if up is not None and up.get("dc") is not None:
            self.lib.calls.append(("fused_normbwd", (up["rec"]["name"], "bwd"), None, None))
        return r

    def wgrad_launch(self, wd, name):
        return tagged(self, (name, "wgrad"), lambda: wg0(self, wd, name))

    for attr, f in (("conv", conv), ("conv_bwd", conv_bwd), ("_wgrad_launch", wgrad_launch)):
        monkeypatch.setattr(Eng, attr, f)


def classify(calls):
    """-> {(layer, op): route} from the tagged launches of one step."""
    from adaptive_voice_conversion_b200 import _lib as L
    by = {}
    for n, tag, a, b in calls:
        if tag is not None:
            by.setdefault(tag, []).append((n, a, b))
    routes = {}
    for (layer, phase), ls in by.items():
        names = [n for n, _, _ in ls]
        if phase == "fwd":
            base = "tc" if "avc_conv_block_tc" in names else "ffma"
            routes[(layer, "fwd")] = base + ("_split" if "avc_norm_apply_fwd" in names else "")
        elif phase == "wgrad":
            routes[(layer, "wgrad")] = {"avc_conv_wgrad_tc": "tc", "avc_conv_wgrad_tc_acc": "tc_acc",
                                        "avc_conv_wgrad": "ffma"}[names[-1]]
        else:
            for n, shuffle, Tout in ls:
                if n == "avc_norm_bwd":
                    routes[(layer, "normbwd")] = "plain_shuffle" if shuffle else ("cached" if Tout <= 128 else "plain")
                elif n == "fused_normbwd":
                    routes[(layer, "normbwd")] = "fused"
            convs = [(n, flags, ts) for n, flags, ts in ls if n in ("avc_conv_block_tc", "avc_conv_block_fwd")]
            if not convs:
                continue                                  # (bank layers: no data gradient)
            n, flags, ts = convs[0]
            if n == "avc_conv_block_tc" and flags & L.F_FOLD:
                r = "tc_fold"
            elif n == "avc_conv_block_tc" and ts == 2:
                r = "tc_s2"
            else:
                r = ("tc" if n == "avc_conv_block_tc" else "ffma") + ("+fold" if "avc_fold_add_fwd" in names else "_direct")
            routes[(layer, "dgrad")] = r
    return routes


def _config(kind):
    return sn_config(80) if kind == "sn" else orc.default_config(80 if kind == "c80" else 512)


def step_routes(monkeypatch, lib, kind, precision, T, env=None, B=2):
    """{(layer, op): route} of one training step of B segments of T frames."""
    with monkeypatch.context() as m:
        for k in ("AVC_FUSED_DENSE", "AVC_FOLD_FUSED", "AVC_NORM_BWD_FUSED", "AVC_WGRAD_ACC"):
            m.delenv(k, raising=False)
        for k, v in (env or {}).items():
            m.setenv(k, v)
        e, P = cpu_engine(m, lib, 132, cfg=_config(kind), precision=precision, stand_in=RouteLib)
        _tagging(m)
        train_step(e, P, B, T)
    assert not e.lib.rejected, e.lib.rejected[:3]
    conv_launches = [c for c in e.lib.calls if c[0] in ("avc_conv_block_tc", "avc_conv_block_fwd", "avc_norm_bwd",
                                                        "avc_norm_apply_fwd", "avc_conv_wgrad", "avc_conv_wgrad_tc")]
    assert all(c[1] is not None for c in conv_launches), [c for c in conv_launches if c[1] is None][:3]
    return classify(e.lib.calls)


def kinds(routes, precision):
    """The routes as (precision, op, route): what a layer-by-layer check has to have seen at least once."""
    return {(precision, op, r) for (_, op), r in routes.items()}


@pytest.fixture(scope="module")
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


@pytest.fixture(scope="module")
def sweep(lib):
    """{(precision, T): routes} for every T of SWEEP, default options."""
    mp = pytest.MonkeyPatch()
    try:
        return {(p, T): step_routes(mp, lib, "c80", p, T) for p in ("fp32", "tf32") for T in SWEEP}
    finally:
        mp.undo()


def test_routes_by_segment_length(sweep, capsys):
    """Every layer has a route for each op it needs, and the routes follow the thresholds of engine.py, csrc/norm.cu
    and csrc/wgrad_tc.cu; the routes each length reaches are listed."""
    first = {}
    for (p, T), routes in sorted(sweep.items()):
        for k in kinds(routes, p):
            first.setdefault(k, T)
        assert routes[("decoder.first_conv_layers.0", "fwd")] in (("tc",) if p == "tf32" else ("ffma",))
        # the content encoder's in_conv: InstanceNorm over T frames, 1 tap
        f = routes[("content_encoder.in_conv_layer", "fwd")]
        assert f == ({"tf32": "tc" if T <= 144 else "tc_split", "fp32": "ffma" if T <= 256 else "ffma_split"}[p]), (p, T, f)
        nb = routes[("content_encoder.first_conv_layers.0", "normbwd")]
        assert nb == ("cached" if T <= 128 else "plain"), (p, T, nb)
        if p == "tf32":
            wg = routes[("content_encoder.first_conv_layers.0", "wgrad")]
            assert wg == ("tc" if T <= 128 else "ffma"), (T, wg)
            wg2 = routes[("content_encoder.second_conv_layers.1", "wgrad")]     # stride 2: Tout = T / 2
            assert wg2 == ("tc" if T <= 128 and T % 16 == 0 else "ffma"), (T, wg2)
            dg = routes[("decoder.first_conv_layers.5", "dgrad")]             # T frames, 5 taps, residual
            assert dg == ("tc_fold" if T + 8 <= 256 else "ffma+fold"), (T, dg)
            s2 = routes[("speaker_encoder.second_conv_layers.1", "dgrad")]     # stride 2 over T frames
            assert s2 == ("tc_s2" if T + 4 <= 512 else "ffma+fold"), (T, s2)
    with capsys.disabled():
        print("\nroutes of a training step, by the shortest segment that reaches them:")
        for k, T in sorted(first.items(), key=lambda kv: (kv[1], kv[0])):
            print(f"  T >= {T:3d}: {k}")


def test_gpu_case_list_reaches_every_route(monkeypatch, lib, sweep, capsys):
    """The union over tests/test_gpu_step_layers.py's TRAIN_CASES reaches every route of the sweep; T = 128 alone
    does not, and what it misses is what the other lengths add."""
    everything = set()
    for (p, T), routes in sweep.items():
        everything |= kinds(routes, p)
    covered, at128 = set(), set()
    with capsys.disabled():
        print("\nroutes per case of test_gpu_step_layers.TRAIN_CASES beyond those of T = 128:")
    base = {p: kinds(sweep[(p, 128)], p) for p in ("fp32", "tf32")}
    for kind, p, B, env, T in TRAIN_CASES:
        ks = kinds(step_routes(monkeypatch, lib, kind, p, T, env), p)
        covered |= ks
        if T == 128:
            at128 |= ks
        extra = sorted(ks - base[p])
        if extra:
            with capsys.disabled():
                print(f"  {kind} {p} B={B} T={T} {env}: {extra}")
    assert sorted(everything - covered) == []
    missing = everything - at128
    assert missing == {("tf32", "fwd", "tc_split"), ("fp32", "fwd", "ffma_split"), ("fp32", "normbwd", "plain"),
                       ("tf32", "normbwd", "plain"), ("tf32", "wgrad", "ffma"), ("tf32", "dgrad", "ffma+fold"),
                       ("tf32", "dgrad", "ffma_direct")}, sorted(missing)


# ------------------------------------------------------------------ segment lengths the decoder reproduces
def test_decoder_length():
    from adaptive_voice_conversion_b200.engine import decoder_length
    cfg = orc.default_config(80)
    assert [decoder_length(cfg, T) for T in (1, 8, 64, 128, 200, 244, 255, 256)] == [8, 8, 64, 128, 200, 248, 256, 256]
    c = dict(cfg, ContentEncoder=dict(cfg["ContentEncoder"], subsample=[1, 2, 1, 2, 1, 1]),
             Decoder=dict(cfg["Decoder"], upsample=[2, 1, 2, 1, 1, 1]))
    assert [decoder_length(c, T) for T in (6, 7, 8)] == [8, 8, 8]
    c["ContentEncoder"]["n_conv_blocks"] = 2          # only the blocks that exist subsample
    assert decoder_length(c, 7) == 16


def _solver_args(tmp_path):
    return types.SimpleNamespace(data_dir="synthetic", train_set="", train_index_file="", logdir=str(tmp_path),
                                 load_model=False, load_opt=False, store_model_path=None, load_model_path=None,
                                 summary_steps=10, save_steps=10, tag="t", iters=0)


@pytest.mark.parametrize("seg", [244, 130, 4])
def test_solver_rejects_a_segment_size_the_decoder_does_not_reproduce(tmp_path, seg):
    """The reconstruction loss pairs the decoder's output with its input frame by frame: a segment_size whose decoded
    length differs is refused when the Solver is built (before any device work), naming segment_size."""
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = orc.default_config(80)
    cfg = dict(cfg, data_loader=dict(cfg["data_loader"], segment_size=seg))
    with pytest.raises(ValueError, match=f"segment_size {seg}"):
        Solver(cfg, _solver_args(tmp_path))


def test_held_out_sets_reject_a_segment_size_the_decoder_does_not_reproduce(tmp_path):
    from adaptive_voice_conversion_b200.evaluate import HeldOut
    cfg = orc.default_config(80)
    cfg = dict(cfg, data_loader=dict(cfg["data_loader"], segment_size=244))
    with pytest.raises(ValueError, match="segment_size 244"):
        HeldOut(["in_test"], str(tmp_path), cfg, device="cpu")


def test_every_trainer_checks_the_segment_length():
    """Speaker adaptation and code fitting step through FusedTrainer.step, which refuses a length the decoder does
    not reproduce before any launch (tests/test_gpu_step_layers.py runs it)."""
    import inspect

    from adaptive_voice_conversion_b200.adapt import AdaptTrainer
    from adaptive_voice_conversion_b200.fit import CodeFitTrainer
    from adaptive_voice_conversion_b200.trainer import FusedTrainer
    assert AdaptTrainer.step is FusedTrainer.step and CodeFitTrainer.step is FusedTrainer.step
    assert "self.step(" in inspect.getsource(CodeFitTrainer.run_step)
    assert "decoder_length" in inspect.getsource(FusedTrainer.step)
