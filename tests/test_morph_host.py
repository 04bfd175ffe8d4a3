"""CPU: the host side of time-varying speaker morphs (AE.inference_morph, Inferencer.inference_morph, inference.py -morph).

* keyframe parsing and speaker_bank.morph_weights against a direct numpy restatement: interpolation, hold before the
  first and after the last keyframe, hard cuts, mixes as keyframes; every error;
* the -morph argument exclusions of inference.py;
* on the fake-library engine of tests/test_conv_tc2_plan.py: a morph decode sends exactly the 12 AdaIN layers through
  avc_norm_apply_morph (decoder.in_conv_layer through avc_norm_apply_varlen), one weight table per layer resolution,
  and a decode without morph issues the same launches with avc_norm_apply_varlen in their place;
* Inferencer.inference_morph rejects bad shapes and weights before anything runs.
"""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

from test_conv_tc2_plan import cpu_engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def root_module(name):
    spec = importlib.util.spec_from_file_location(f"_root_{name}", os.path.join(ROOT, f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


# ----------------------------------------------------------------------------- keyframes
def reference_weights(keyframes, n, fps):
    """Frame by frame, with plain loops."""
    names = []
    for spec, _ in keyframes:
        for part in spec.split(","):
            nm = part.split(":")[0]
            if nm not in names:
                names.append(nm)
    vecs = []
    for spec, _ in keyframes:
        v = np.zeros(len(names))
        for part in spec.split(","):
            nm, _, w = part.partition(":")
            v[names.index(nm)] = float(w) if w else 1.0
        vecs.append(v / v.sum())
    times = [float(t) for _, t in keyframes]
    out = np.zeros((len(names), n))
    for f in range(n):
        s = f / fps
        if s < times[0]:
            out[:, f] = vecs[0]
            continue
        last = max(i for i, t in enumerate(times) if t <= s)
        if last == len(times) - 1:
            out[:, f] = vecs[-1]
        else:
            a = (s - times[last]) / (times[last + 1] - times[last])
            out[:, f] = (1 - a) * vecs[last] + a * vecs[last + 1]
    return names, out.astype(np.float32)


@pytest.mark.parametrize("keyframes", [
    [("p225", 0.0)],                                                              # one speaker throughout
    [("p225", 0.5), ("p226", 1.0)],                                               # hold, glide, hold
    [("p225", 0.0), ("p225", 0.4), ("p226", 0.45), ("p226", 0.9), ("p225:0.5,p226:0.5", 1.2)],
    [("p225", 0.3), ("p226", 0.3), ("p227:3,p225:1", 0.3), ("p226", 0.8)],       # hard cuts at one time
    [("p225:2,p226:6", 0.0), ("p227", 0.7), ("p226:1,p225:1,p227:2", 2.5)],       # mixes, the last past the end
])
def test_morph_weights_match_a_direct_restatement(keyframes):
    from adaptive_voice_conversion_b200.speaker_bank import morph_weights
    for n, fps in ((1, 80.0), (97, 80.0), (130, 100.0)):
        names, w = morph_weights(keyframes, n, fps)
        rn, rw = reference_weights(keyframes, n, fps)
        assert names == rn and w.dtype == np.float32 and w.shape == (len(rn), n)
        np.testing.assert_allclose(w, rw, rtol=0, atol=2e-7)
        np.testing.assert_allclose(w.astype(np.float64).sum(0), 1.0, atol=1e-6)


def test_morph_weights_hard_cut_and_hold():
    from adaptive_voice_conversion_b200.speaker_bank import morph_weights
    names, w = morph_weights([("a", 0.1), ("b", 0.1)], 20, 80)     # frame 8 lies at 0.1 s
    assert names == ["a", "b"]
    assert (w[0, :8] == 1).all() and (w[1, 8:] == 1).all() and (w[0, 8:] == 0).all()


def test_parse_keyframe_and_errors():
    from adaptive_voice_conversion_b200.speaker_bank import morph_weights, parse_keyframe
    assert parse_keyframe("p225@0") == ("p225", 0.0)
    assert parse_keyframe("p225:0.5,p226:0.5@12") == ("p225:0.5,p226:0.5", 12.0)
    for bad, msg in (("p225", "SPEC@SECONDS"), ("p225@abc", "not a number"), ("p225@-1", ">= 0"), ("p225@nan", ">= 0"),
                     ("@3", "expected .NAME"), ("p225,p225@1", "twice"), ("p225:x@1", "not a number"), ("p225:-1@1", ">= 0")):
        with pytest.raises(ValueError, match=msg):
            parse_keyframe(bad)
    with pytest.raises(ValueError, match="no keyframes"):
        morph_weights([], 10, 80)
    with pytest.raises(ValueError, match="must not decrease"):
        morph_weights([("a", 1.0), ("b", 0.5)], 10, 80)
    with pytest.raises(ValueError, match=">= 0"):
        morph_weights([("a", -0.5)], 10, 80)
    with pytest.raises(ValueError, match="twice"):
        morph_weights([("a,b,a", 0.0)], 10, 80)


def test_morph_table_names_bank_rows():
    from adaptive_voice_conversion_b200.speaker_bank import SpeakerBank, morph_table
    codes = torch.arange(12, dtype=torch.float32).view(3, 4)
    bank = SpeakerBank(["p1", "p2", "p3"], codes, [1, 1, 1], [["u1"], ["u2"], ["u3"]], "fp")
    c, w = morph_table(bank, [("p3", 0), ("p1:1,p3:1", 1)], 90, 80)
    assert torch.equal(c, codes[[2, 0]]) and w.shape == (2, 90) and w.dtype == torch.float32
    with pytest.raises(ValueError, match="not in the bank"):
        morph_table(bank, [("p9", 0)], 10, 80)


def test_inference_cli_morph_argument_errors():
    inf = root_module("inference")
    p = inf.parser()
    base = ["-s", "a", "-o", "b"]
    for argv, msg in ((base + ["-morph", "p1@0"], "needs -bank"),
                      (base + ["-bank", "k", "-morph", "p1@0", "-t", "x"], "excludes"),
                      (base + ["-bank", "k", "-morph", "p1@0", "-speaker", "p1"], "excludes"),
                      (["-pairs", "f", "-o", "d", "-bank", "k", "-morph", "p1@0"], "excludes"),
                      (base + ["-bank", "k", "-morph", "p1@1", "p2@0.5"], "must not decrease"),
                      (base + ["-bank", "k", "-morph", "p1@x"], "not a number"),
                      (base + ["-bank", "k", "-morph", "p1"], "SPEC@SECONDS")):
        with pytest.raises(SystemExit):
            inf.check_args(p, p.parse_args(argv))
    args = p.parse_args(base + ["-bank", "k", "-morph", "p1@0", "p1@4", "p2@4.3", "p1:0.5,p2:0.5@12"])
    inf.check_args(p, args)
    assert args.keyframes == [("p1", 0.0), ("p1", 4.0), ("p2", 4.3), ("p1:0.5,p2:0.5", 12.0)]


# ----------------------------------------------------------------------------- what the engine launches
class CallLog:
    """Wraps the fake library of cpu_engine: logs every call as (name, detail)."""

    def __init__(self, inner):
        self.inner, self.calls = inner, []

    def __getattr__(self, name):
        fn = getattr(self.inner, name)

        def f(*a):
            detail = None
            if name in ("avc_norm_apply_varlen", "avc_norm_apply_morph"):
                d = a[0]._obj
                detail = (d.Tout * (1 + d.shuffle), a[2], a[3], bool(d.cond))
                if name == "avc_norm_apply_morph":
                    detail += (a[5], a[6])
            elif name == "avc_morph_weights":
                detail = (a[2], a[3], a[4], a[5], a[7])
            self.calls.append((name, detail))
            return fn(*a)
        return f


def decode(e, P, B, T, morph):
    from adaptive_voice_conversion_b200.engine import A4, Lengths, varlen_extent
    Te = varlen_extent(e.cfg, T, source=True)
    z4 = A4.empty(B, e.cfg["Decoder"]["c_in"], Te // 8, e.dev)
    lens = Lengths(torch.full((B,), T, dtype=torch.int32), 8, 1)
    with torch.no_grad():
        return e.decoder_fwd(P, z4, None if morph else torch.empty(B, e.cfg["SpeakerEncoder"]["c_out"]), False, lens=lens,
                             morph=morph)[0]


@pytest.mark.parametrize("c_in", (80, 512))
def test_morph_decode_launches(monkeypatch, lib, c_in):
    e, P = cpu_engine(monkeypatch, lib, 132, c_in)
    log = CallLog(e.lib)
    e.lib = log
    B, T, K = 4, 203, 3
    c_out = e.cfg["SpeakerEncoder"]["c_out"]
    dec_m = decode(e, P, B, T, (torch.empty(B, K, c_out), torch.empty(B, K, T)))
    with_morph = list(log.calls)
    log.calls.clear()
    dec_p = decode(e, P, B, T, None)
    plain = list(log.calls)
    assert (dec_m.C, dec_m.T) == (dec_p.C, dec_p.T)
    morph = [c for c in with_morph if c[0] == "avc_norm_apply_morph"]
    varlen = [c for c in with_morph if c[0] == "avc_norm_apply_varlen"]
    nblk = e.cfg["Decoder"]["n_conv_blocks"]
    assert len(morph) == 2 * nblk == 12 and all(d[3] and d[4] == K for _, d in morph)
    assert len(varlen) == 1 and not varlen[0][1][3]                     # in_conv_layer: InstanceNorm, no AdaIN
    # the anchor rows of one sample: [K, 2n, 2 c_h] -> K rows 2n * 2 c_h floats apart
    assert all(d[5] == 2 * nblk * 2 * e.cfg["Decoder"]["c_h"] for _, d in morph)
    # one weight table per layer resolution f, each as long as the layers that read it
    Tdec = dec_m.T
    tables = [d for n, d in with_morph if n == "avc_morph_weights"]
    assert sorted(d[3] for d in tables) == [1, 2, 4, 8] and all(d[:3] == (B, K, T) and d[4] == Tdec // d[3] for d in tables)
    assert sorted({d[0] for _, d in morph}) == sorted(Tdec // d[3] for d in tables)
    # without morph: the same launches, avc_norm_apply_varlen where the morph has avc_norm_apply_morph
    assert not any(n in ("avc_norm_apply_morph", "avc_morph_weights") for n, _ in plain)
    strip = [(n if n != "avc_norm_apply_morph" else "avc_norm_apply_varlen") for n, _ in with_morph if n != "avc_morph_weights"]
    assert strip == [n for n, _ in plain]
    assert [d[:3] for n, d in with_morph if n == "avc_norm_apply_morph"] == \
        [d[:3] for n, d in plain if n == "avc_norm_apply_varlen" and d[3]]


def test_morph_decode_needs_padded_inference(monkeypatch, lib):
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200.engine import A4
    e, P = cpu_engine(monkeypatch, lib, 132, 80)
    z4 = A4.empty(2, e.cfg["Decoder"]["c_in"], 16, e.dev)
    with pytest.raises(L.AvcError, match="morph needs lens"):
        e.decoder_fwd(P, z4, None, False, morph=(torch.empty(2, 1, 128), torch.empty(2, 1, 128)))


# ----------------------------------------------------------------------------- Inferencer input validation
def fake_inferencer():
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.inference import Inferencer
    inf = object.__new__(Inferencer)
    inf.config = orc.default_config(80)
    inf.config["data_loader"] = {"frame_size": 1}

    def boom(*a, **k):
        raise AssertionError("nothing may run before the inputs are validated")
    inf.model = types.SimpleNamespace(inference_morph=boom, engine=boom)
    inf._morph_slot = boom
    return inf


def test_inferencer_morph_rejects_bad_inputs_before_running():
    inf = fake_inferencer()
    x = torch.zeros(100, 80)
    c = torch.zeros(2, 128)
    w = torch.ones(2, 100)
    cases = [
        (([x], [c], [w, w]), "same length"),
        (([x], [torch.zeros(2, 64)], [w]), "expected codes"),
        (([x], [torch.zeros(65, 128)], [torch.ones(65, 100)]), "expected codes"),
        (([x], [c], [torch.ones(2, 99)]), "expected codes"),
        (([x], [c.double()], [w]), "float32"),
        (([x], [c], [torch.tensor([[1.0] * 100, [-1.0] + [0.0] * 99])]), "positive sum"),
        (([x], [c], [torch.zeros(2, 100)]), "positive sum"),
        (([x], [c], [torch.full((2, 100), float("nan"))]), "positive sum"),
        (([x], [c], [torch.full((2, 100), float("inf"))]), "positive sum"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError, match=msg):
            inf.inference_morph(*args)
    assert inf.inference_morph([], [], []) == []
    with pytest.raises(ValueError, match="source frames"):          # shorter than the model accepts
        inf.inference_morph([torch.zeros(3, 80)], [c], [torch.ones(2, 3)])
