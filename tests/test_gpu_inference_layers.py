"""GPU: every layer of padded-batch inference, of grouped speaker codes, and of unpadded inference at c512 and with
spectral norm, against tests/_layer_ref.py's float64 restatement, on the engine's own inputs to each layer (the hooks
and the tap of test_gpu_step_layers.py).

A padded batch is checked one sample at a time.  The reference runs on sample b's valid frames alone; at each
boundary the tap compares it with the engine's value of sample b, cut to the frames the reference has, and continues
with the engine's.  The reference pads by reflection at its own last frame and never sees the frames past it, so a halo
frame the engine reflected from the wrong place, InstanceNorm statistics over one frame too many or too few, or a POOL
residual that averages the wrong frames is an error at the layer that has it.  At every layer the reference's length
must also be the valid length the engine's Lengths give that layer (what avc_varlen_tail, avc_norm_apply_varlen and the
time means read), so the reference's geometry checks the engine's length bookkeeping.

- The padding of the inputs holds NaN in one call and +-1e4 noise in another: the outputs are the same bits, and so
  is the instrumented call's.
- Every conv layer is checked for every sample, and every conv-family launch (with avc_norm_apply_varlen and
  avc_varlen_tail) belongs to a checked layer.
- Grouped codes: every member's conv layers as above, then each set's pooled row against the float64 mean over its
  members' valid last-layer frames together, and its code against the dense stack of that row.
- Spectral norm: the model is in eval(), as a converter runs it; W_bar is checked against the float64 restatement
  without a power iteration, then feeds the chain.
"""
import types

import pytest
import torch

import _layer_ref as LR
from test_gpu_step_layers import (CONV_FAMILY, INFER_CASES, Capture, Checker, _report, eval_wbar, inference_layers,
                                  inference_model, install)

pytestmark = pytest.mark.gpu

FAMILY = CONV_FAMILY + ("avc_norm_apply_varlen", "avc_varlen_tail")
# Padded batches and grouped codes: about 3x the worst measured on 1x H100 80GB HBM3 (700 W power limit), over every
# padded and grouped case of this file:
#   fp32: fwd 5.6e-6 (c512 decoder.in_conv_layer, the 17-frame source), misc 6.7e-7 (sn, an AdaIN row)
#   tf32: fwd 7.2e-6 (c512 speaker_encoder.conv_bank.7, the 1000-frame member), misc 6.3e-7 (sn, an AdaIN row)
# Every InstanceNorm layer of a padded batch runs as a plain conv + the two-pass avc_norm_apply_varlen, so a short
# sample needs no allowance for the fused tensor-core epilogue's one-pass variance (test_inference_layers' 1.2e-3):
# in TF32 the 17-frame source, whose decoder in_conv normalises 3 frames, stays below the worst above.
# ambiguous ReLU elements per padded batch (8 pairs): 191-218; per grouped call (12 members): 99-116.
# The unpadded c512 and sn cases keep test_gpu_step_layers.TOL: measured fwd 1.1e-5 fp32 (c512, 17 frames), 1.2e-5 tf32
# (sn, 1000 frames), misc 7.2e-7; the 17-frame TF32 cases keep the one-pass-variance allowance (c512 5.5e-5, sn 1.6e-4).
TOL_PADDED = {"fp32": dict(fwd=1.7e-5, misc=2e-6), "tf32": dict(fwd=2.2e-5, misc=2e-6)}
# 8 pairs: the minimum lengths (mcd.min_frames), lengths odd at every subsampling level (273; 49, 337), the boundaries
# of the unpadded fused kernels (128, 129, 144, 145), lengths the persistent kernel time-tiles (>= 600), and a length
# equal to the batch's extent (1000 source, 600 reference frames)
SRC_LENS = [17, 273, 128, 129, 144, 145, 601, 1000]
REF_LENS = [9, 49, 145, 144, 129, 128, 337, 600]
# grouped codes: sets of 1, 3, 2, 1 and 5 reference utterances
GROUP_SIZES = [1, 3, 2, 1, 5]
GROUP_LENS = [9, 600, 49, 128, 129, 145, 144, 337, 17, 81, 1000, 33]


def _frames(rec, b):
    t, div, mul = rec
    return -(-int(t[b]) // div) * mul


class SampleChecker(Checker):
    """The tap for sample b of a padded batch: each captured value is cut to sample b and to the frames the reference
    has, after checking that length against the engine's Lengths.  n: the sample's input frames per stack."""

    def __init__(self, cap, cfg, tf32, b, n_src, n_ref):
        super().__init__(cap, {}, cfg, tf32)
        self.full, self.b = cap, b
        self.n = dict(speaker_encoder=n_ref, content_encoder=n_src, decoder=n_src)
        self.last_content = f"content_encoder.second_conv_layers.{cfg['ContentEncoder']['n_conv_blocks'] - 1}"
        self.layers = set()

    def valid(self, name, where):
        """The engine's valid frames of sample b at the input ("x") or the output ("out") of layer name."""
        f = self.full.fwd[name]
        if f["lens"] is None:      # the content heads (K = 1) read the content encoder's last layer as it left it
            return self.valid(self.last_content, "out")
        t = f["lens"][0]
        if int(t[self.b]) != self.n[name.split(".")[0]]:
            self.problems.append(f"{name}: the engine's length of sample {self.b} is {int(t[self.b])}, not "
                                 f"{self.n[name.split('.')[0]]}")
        if where == "x":
            return _frames(f["lens"], self.b)
        return _frames(f["lens_out"], self.b) * (2 if f["shuffle"] else 1)

    def _length(self, what, ref_n, eng_n):
        if ref_n != eng_n:
            self.problems.append(f"{what}: sample {self.b} has {ref_n} frames, the engine's Lengths give {eng_n}")

    def __call__(self, kind, name, ref, **info):
        full, b = self.full, self.b
        fwd = {}
        if kind == "out":
            self._length(name, ref.shape[2], self.valid(name, "out"))
            f = full.fwd[name]
            fwd[name] = dict(f, x=f["x"][b:b + 1, :, :self.valid(name, "x")], out=f["out"][b:b + 1, :, :ref.shape[2]])
            self.layers.add(name)
        elif kind in ("x", "z"):
            layer = name + ".conv_bank.0" if kind == "x" else "decoder.in_conv_layer"
            self._length(layer + " input", ref.shape[2], self.valid(layer, "x"))
            f = full.fwd[layer]
            fwd[layer] = dict(f, x=f["x"][b:b + 1, :, :ref.shape[2]])
        elif kind == "conds":
            fwd = {n: dict(f, cond=f["cond"][b:b + 1]) for n, f in full.fwd.items() if f["cond"] is not None}
        self.cap = types.SimpleNamespace(fwd=fwd, emb=None if full.emb is None else full.emb[b:b + 1])
        return super().__call__(kind, name, ref, **info)


def merge(total, chk, tag):
    """Fold one sample's checker into the case's: the worst per kind (named by layer and sample), the problems."""
    for k, v in chk.worst.items():
        total.err(k, f"{chk.where[k]} [{tag}]", v)
    total.amb += chk.amb
    total.problems += chk.problems


def stray(launches, checked):
    """Conv-family launches that belong to no checked layer.  A varlen tail launched between layers belongs to the
    layer that reads it next (the bank convs' shared reflection, a POOL residual's replicated frame), one after the
    last layer to that layer (the zeroed tail of the decoder output).  So a tail launched in the wrong place is not
    stray here: it shows only in the values of the layer that reads it."""
    out, pending, last = [], [], None
    for n, t in launches:
        if n not in FAMILY:
            continue
        if t is None and n == "avc_varlen_tail":
            pending.append((n, t))
            continue
        if t is None or t[0] not in checked:
            out.append((n, t))
        else:
            last = t[0]
        pending = []
    return out + (pending if last is None else [])


def padded(us, T, fill, seed=1):
    """The utterances [C, n] in a [B, C, T] batch whose padding holds NaN or +-1e4 noise."""
    if fill == "nan":
        out = torch.full((len(us), us[0].shape[0], T), float("nan"))
    else:
        out = 1e4 * (2 * torch.rand((len(us), us[0].shape[0], T), generator=torch.Generator().manual_seed(seed)) - 1)
    for b, u in enumerate(us):
        out[b, :, :u.shape[1]] = u
    return out.cuda()


def utterances(n_mels, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn((n_mels, n), generator=g) for n in lens]


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def check_bounds(total, precision):
    assert not total.problems, total.problems[:10]
    tol = TOL_PADDED[precision]
    bad = {k: (v, total.where[k]) for k, v in total.worst.items() if not v <= tol[k]}
    assert not bad, bad


PADDED_CASES = [(k, p) for k in ("c80", "c512", "sn") for p in ("fp32", "tf32")]


@pytest.mark.parametrize("kind,precision", PADDED_CASES, ids=[f"{k}-{p}" for k, p in PADDED_CASES])
def test_padded_inference_layers(monkeypatch, kind, precision):
    monkeypatch.setenv("AVC_PRECISION", precision)
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    m, cfg = inference_model(kind)
    n_mels = cfg["SpeakerEncoder"]["c_in"]
    xs, cs = utterances(n_mels, SRC_LENS, 0), utterances(n_mels, REF_LENS, 1)
    T, T_c = max(SRC_LENS), max(REF_LENS)
    lx, lc = torch.tensor(SRC_LENS), torch.tensor(REF_LENS).cuda()

    def run(fill):
        with torch.no_grad():
            return m.inference(padded(xs, T, fill), padded(cs, T_c, fill), lengths=lx, cond_lengths=lc)
    nan, noise = run("nan"), run("noise")
    eng = m.engine(nan.device)
    cap = Capture()
    install(monkeypatch, eng, cap)
    dec = run("noise")
    torch.cuda.synchronize()
    eng.check_tc_status()

    tf32 = precision == "tf32"
    total = Checker(cap, {}, cfg, tf32)
    P = dict(m.named_parameters())
    assert set(cap.wbar) == set(eng.sn_names())
    P.update(eval_wbar(m, cap, total))
    layers = set(eng.conv_names())
    for b, (n, n_c) in enumerate(zip(SRC_LENS, REF_LENS)):
        chk = SampleChecker(cap, cfg, tf32, b, n, n_c)
        ref, _ = LR.ae_inference(P, cfg, xs[b][None].cuda(), cs[b][None].cuda(), chk, cap.tc)
        To = 8 * -(-n // 8)
        assert ref.shape[2] == To
        chk.err("misc", "dec", Checker._rel(dec[b:b + 1, :, :To], ref, ref.abs().max()))
        assert bool((dec[b, :, To:] == 0).all()), f"sample {b}: the output past its valid frames is not 0"
        assert chk.layers == layers, (b, sorted(layers ^ chk.layers))
        merge(total, chk, f"b={b} n={n} n_c={n_c}")
    _report(f"padded {kind} {precision}", total)
    assert not stray(cap.launches, layers), stray(cap.launches, layers)[:5]
    check_bounds(total, precision)     # (first: it names the layer a padding-dependent value comes from)
    assert same_bits(nan, noise), "the padding's content changed the output"
    assert same_bits(dec, noise), "the instrumented call changed the output"


GROUP_CASES = [(k, p) for k in ("c80", "c512") for p in ("fp32", "tf32")]


@pytest.mark.parametrize("kind,precision", GROUP_CASES, ids=[f"{k}-{p}" for k, p in GROUP_CASES])
def test_grouped_speaker_code_layers(monkeypatch, kind, precision):
    from adaptive_voice_conversion_b200 import engine as E
    monkeypatch.setenv("AVC_PRECISION", precision)
    m, cfg = inference_model(kind)
    cs = utterances(cfg["SpeakerEncoder"]["c_in"], GROUP_LENS, 2)
    T = max(GROUP_LENS)
    lc = torch.tensor(GROUP_LENS).cuda()
    offs = torch.tensor([0] + GROUP_SIZES).cumsum(0)

    def run(fill):
        with torch.no_grad():
            return m.get_speaker_embeddings(padded(cs, T, fill), lengths=lc, groups=offs)
    nan, noise = run("nan"), run("noise")
    assert nan.shape == (len(GROUP_SIZES), cfg["SpeakerEncoder"]["c_out"])
    eng = m.engine(nan.device)
    cap = Capture()
    install(monkeypatch, eng, cap)
    dense0 = E.Engine._speaker_dense

    def speaker_dense(self, P, pooled, train, ctx):
        cap.pooled = pooled.clone()
        return dense0(self, P, pooled, train, ctx)
    monkeypatch.setattr(E.Engine, "_speaker_dense", speaker_dense)
    codes = run("noise")
    torch.cuda.synchronize()
    eng.check_tc_status()

    tf32 = precision == "tf32"
    total = Checker(cap, {}, cfg, tf32)
    P = dict(m.named_parameters())
    layers = {n for n in eng.conv_names() if n.startswith("speaker_encoder.")}
    last = []
    for b, n in enumerate(GROUP_LENS):
        chk = SampleChecker(cap, cfg, tf32, b, None, n)
        last.append(LR.speaker_convs(P, cfg, cs[b][None].cuda(), chk, cap.tc))
        assert chk.layers == layers, (b, sorted(layers ^ chk.layers))
        merge(total, chk, f"member {b} n={n}")
    for g in range(len(GROUP_SIZES)):
        o0, o1 = int(offs[g]), int(offs[g + 1])
        row = torch.cat(last[o0:o1], dim=2).double().mean(dim=2)
        total.err("misc", f"pooled[{g}]", Checker._rel(cap.pooled[g:g + 1], row, row.abs().max()))
        code = LR.dense_pooled(P, cfg, cap.pooled[g:g + 1])
        total.err("misc", f"code[{g}]", Checker._rel(codes[g:g + 1], code, code.abs().max()))
    _report(f"grouped {kind} {precision}", total)
    assert not stray(cap.launches, layers), stray(cap.launches, layers)[:5]
    check_bounds(total, precision)
    assert same_bits(nan, noise), "the padding's content changed the codes"
    assert same_bits(codes, noise), "the instrumented call changed the codes"


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("T,T_c", INFER_CASES)
@pytest.mark.parametrize("kind", ["c512", "sn"])
def test_unpadded_inference_layers(monkeypatch, kind, precision, T, T_c):
    inference_layers(monkeypatch, kind, precision, T, T_c)
