"""GPU: padded batches of different-length utterances (AE.inference / get_speaker_embeddings with lengths,
Inferencer.inference_padded, inference.py -pairs) and their kernels (avc_norm_apply_varlen,
avc_time_mean_varlen_fwd, avc_varlen_tail).

* each sample of a padded batch is its unpadded conversion within twice the bound test_gpu_model.py's ragged test uses
  (TOL_FP32, TOL_TF32 below), three pairs also within that test's bound of the float64 oracle; the tail is exactly 0;
* the padding's content (zeros, noise, NaN) never changes a valid bit; permuting the batch permutes the outputs;
* lengths=None is the unchanged path: the same launches, the same bits;
* the kernels against a float64 restatement on identical inputs, with sentinels outside every written region;
* inference_padded against inference_ragged, graph replay against eager, and no capture on a second call in the grid;
* the -pairs CLI against the single-pair CLI on seeded synthetic wavs.
"""
import os
import subprocess
import sys
import types
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from _norm_ref import RES_POOL, RES_SAME, RES_UP, from_a4, norm_apply, to_a4
from _sn_ref import sn_config

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 1e-3
# Against the unpadded call: twice the bound of test_gpu_model.py's inference_ragged test (1e-5 fp32, 2e-3 TF32).  That
# test's buckets run the very kernels of the stand-alone call; a padded batch runs every InstanceNorm layer as a plain
# conv + avc_norm_apply_varlen where the stand-alone call fuses the short ones (<= 144 columns) with another summation
# order, and a 17-frame source normalises 3 latent frames per channel, which amplifies that rounding past 1e-5 in fp32.
# The float64 oracle check (REL / 8e-3, as in the ragged test) is the accuracy contract.
TOL_FP32, TOL_TF32 = 2e-5, 4e-3
SENTINEL = -7777.0
SRC_LENS = [17, 600, 101, 128, 129, 144, 145, 301]          # + the extent itself below
REF_LENS = [9, 33, 600, 145, 128, 77, 301, 129]


@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


def tol(precision, fp32, tf32):
    return fp32 if precision == "fp32" else tf32


def relerr(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def make_model(cfg):
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(0)
    m = AE(cfg)                        # Decoder.sn: torch's default init, with its u and v
    if not cfg["Decoder"].get("sn", False):
        m.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    return m.cuda().eval()


def utterances(n_mels, src_lens, ref_lens, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn((n_mels, t), generator=g) for t in src_lens]
    cs = [torch.randn((n_mels, t), generator=g) for t in ref_lens]
    return xs, cs


def padded(us, T, fill="zeros", seed=1):
    g = torch.Generator().manual_seed(seed)
    out = torch.zeros(len(us), us[0].shape[0], T)
    if fill == "noise":
        out = 100 * torch.randn(out.shape, generator=g)
    elif fill == "nan":
        out[:] = float("nan")
        out[0, :, -1] = float("inf")
    for b, u in enumerate(us):
        out[b, :, :u.shape[1]] = u
    return out.cuda()


CONFIGS = {"c80": lambda: orc.default_config(80), "c512": lambda: orc.default_config(512), "sn": lambda: sn_config(80)}


@pytest.mark.parametrize("cfg_name", list(CONFIGS))
def test_padded_batch_equals_per_utterance(precision, cfg_name):
    cfg = CONFIGS[cfg_name]()
    m = make_model(cfg)
    n_mels = cfg["SpeakerEncoder"]["c_in"]
    T, Tc = 608, 608
    src = SRC_LENS + [T]
    ref = REF_LENS + [Tc]
    xs, cs = utterances(n_mels, src, ref)
    lx, lc = torch.tensor(src), torch.tensor(ref).cuda()
    with torch.no_grad():
        dec = m.inference(padded(xs, T), padded(cs, Tc), lengths=lx, cond_lengths=lc)
        emb = m.get_speaker_embeddings(padded(cs, Tc), lengths=lc)
    assert dec.shape == (len(src), n_mels, T)
    for b, (x, c) in enumerate(zip(xs, cs)):
        To = 8 * -(-src[b] // 8)
        with torch.no_grad():
            alone = m.inference(x[None].cuda(), c[None].cuda())
            e1 = m.get_speaker_embeddings(c[None].cuda())
        assert relerr(dec[b, :, :To], alone[0]) < tol(precision, TOL_FP32, TOL_TF32), (b, src[b], ref[b])
        assert relerr(emb[b], e1[0]) < tol(precision, TOL_FP32, TOL_TF32), (b, ref[b])
        assert bool((dec[b, :, To:] == 0).all()), b
        # the oracle at typical lengths; a 17-frame source normalises 3 latent frames per channel, where TF32 rounding
        # alone moves the stand-alone call by about the bound
        if cfg_name == "c80" and b in (2, 6, 8):
            with torch.no_grad():
                r = orc.ae_inference(orc.init_state(cfg, 0), cfg, x[None], c[None])
            assert relerr(dec[b, :, :To], r) < tol(precision, REL, 8e-3), b
    m.engine("cuda:0").check_tc_status()


def test_padding_content_and_order_do_not_matter(precision):
    cfg = orc.default_config(80)
    m = make_model(cfg)
    xs, cs = utterances(80, SRC_LENS, REF_LENS, seed=3)
    lx, lc = torch.tensor(SRC_LENS).cuda(), torch.tensor(REF_LENS).cuda()
    res = {}
    with torch.no_grad():
        for fill in ("zeros", "noise", "nan"):
            res[fill] = (m.inference(padded(xs, 600, fill), padded(cs, 640, fill), lengths=lx, cond_lengths=lc),
                         m.get_speaker_embeddings(padded(cs, 640, fill), lengths=lc))
        perm = [5, 2, 7, 0, 3, 1, 6, 4]
        dp = m.inference(padded([xs[i] for i in perm], 600, "noise"), padded([cs[i] for i in perm], 640, "nan"),
                         lengths=lx[perm], cond_lengths=lc[perm])
    for fill in ("noise", "nan"):
        assert torch.equal(res[fill][0], res["zeros"][0]), fill
        assert torch.equal(res[fill][1], res["zeros"][1]), fill
    assert torch.isfinite(res["nan"][0]).all()
    assert torch.equal(dp, res["zeros"][0][perm])


def test_lengths_none_is_the_unchanged_path(precision):
    from adaptive_voice_conversion_b200 import _lib as L
    cfg = orc.default_config(80)
    m = make_model(cfg)
    g = torch.Generator().manual_seed(5)
    x, c = torch.randn((3, 80, 200), generator=g).cuda(), torch.randn((3, 80, 150), generator=g).cuda()
    with torch.no_grad():
        m.inference(x, c)                              # weight packs
        torch.cuda.synchronize()
        n0 = L.launch_count()
        a = m.inference(x, c)
        torch.cuda.synchronize()
        n1 = L.launch_count()
        b = m.inference(x, c, lengths=None, cond_lengths=None)
        torch.cuda.synchronize()
        n2 = L.launch_count()
        e1, e2 = m.get_speaker_embeddings(c), m.get_speaker_embeddings(c, lengths=None)
    assert n2 - n1 == n1 - n0
    assert torch.equal(a, b) and torch.equal(e1, e2)
    # and invalid lengths raise before any launch
    n3 = L.launch_count()
    for kw in (dict(lengths=torch.tensor([16, 200, 200])), dict(lengths=torch.tensor([17, 201, 200])),
               dict(cond_lengths=torch.tensor([8, 9, 9])), dict(lengths=torch.tensor([17, 17])),
               dict(lengths=torch.tensor([17.0, 17.0, 17.0]))):
        with pytest.raises(L.AvcError):
            m.inference(x, c, **kw)
    with pytest.raises(L.AvcError):
        m(x, lengths=torch.tensor([200, 200, 200]))
    assert L.launch_count() == n3


# ------------------------------------------------------------------ the kernels against float64
@pytest.mark.parametrize("shuffle,res_mode", [(False, 0), (False, RES_SAME), (False, RES_POOL), (True, 0), (True, RES_UP)])
@pytest.mark.parametrize("cond,relu", [(False, True), (True, True), (True, False)])
def test_norm_apply_varlen_kernel(shuffle, res_mode, cond, relu):
    from adaptive_voice_conversion_b200 import _lib as L
    g = torch.Generator().manual_seed(7)
    B, Co, T, div = 8, 16, 150, 2 if res_mode == RES_POOL else 1     # POOL: the block input is one stride-2 level up
    lens = [1, 2, 33, 75, 149, 300, 299, 151] if div == 2 else [1, 2, 33, 75, 149, 150, 99, 150]
    Cn, Tn = (Co // 2, 2 * T) if shuffle else (Co, T)
    c = torch.randn((B, Co, T), generator=g) * 3 + 1
    c[0, 0] = 2.5                                                     # a constant channel
    cond_t = torch.randn((B, 2 * Cn), generator=g) if cond else None
    res_T = {0: 1, RES_SAME: Tn, RES_POOL: 2 * T, RES_UP: T}[res_mode]
    res = torch.randn((B, Cn, res_T), generator=g)
    out, ca, ra = torch.full((B, Cn // 4, Tn, 4), SENTINEL, device="cuda"), to_a4(c), to_a4(res)
    cv, lt = cond_t.cuda() if cond else None, torch.tensor(lens, dtype=torch.int32).cuda()
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups, d.Tin, d.Tout = B, 4, Co, 1, 1, 1, T, T
    d.shuffle, d.norm, d.relu, d.eps = int(shuffle), 1, int(relu), 1e-5
    d.save_c, d.out, d.out_bstride = ca.data_ptr(), out.data_ptr(), out[0].numel()
    if cond:
        d.cond, d.cond_bstride = cv.data_ptr(), cv.stride(0)
    if res_mode:
        d.res, d.res_bstride, d.res_mode, d.res_T = ra.data_ptr(), ra[0].numel(), res_mode, res_T
    assert L.load().avc_norm_apply_varlen(C.byref(d), lt.data_ptr(), div, 1, None) == 0, L.last_error()
    got = from_a4(out)
    for b in range(B):
        Lb = -(-lens[b] // div)
        Ln = 2 * Lb if shuffle else Lb
        r = res[b:b + 1, :, :{0: 0, RES_SAME: Ln, RES_POOL: lens[b], RES_UP: Lb}[res_mode]] if res_mode else None
        ref, _, _ = norm_apply(c[b:b + 1, :, :Lb], shuffle=shuffle, norm=True, cond=cond_t[b:b + 1] if cond else None,
                               relu=relu, res=r, res_mode=res_mode)
        assert relerr(got[b:b + 1, :, :Ln], ref) < 5e-6, b
        assert bool((got[b, :, Ln:] == SENTINEL).all()), b


def test_time_mean_varlen_and_tail_kernels():
    """On channels [4, 12) of a 16-channel tensor, lengths ceil(L / 2) of L = 1 2 7 39 40 79."""
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    x = torch.randn((6, 16, 40), generator=torch.Generator().manual_seed(9))
    B, T, c0, Cc = 6, 40, 4, 8
    lens = [1, 2, 7, 39, 40, 79]
    Lb = [-(-v // 2) for v in lens]
    lt = torch.tensor(lens, dtype=torch.int32).cuda()
    xa = to_a4(x)
    mean = torch.full((B * Cc + 4,), SENTINEL, device="cuda")
    assert lib.avc_time_mean_varlen_fwd(xa[:, 1:3].data_ptr(), xa[0].numel(), mean.data_ptr(), B, Cc, T, lt.data_ptr(), 2, 1,
                                        None) == 0
    for b in range(B):
        assert relerr(mean[b * Cc:(b + 1) * Cc], x[b, c0:c0 + Cc, :Lb[b]].double().mean(dim=1)) < 2e-6, b
    assert bool((mean[B * Cc:] == SENTINEL).all())
    for mode, n in ((L.TAIL_REFLECT, 3), (L.TAIL_REPLICATE, 1), (L.TAIL_ZERO, 1)):
        xa = to_a4(x)
        assert lib.avc_varlen_tail(xa[:, 1:3].data_ptr(), xa[0].numel(), B, Cc, T, lt.data_ptr(), 2, 1, mode, n, None) == 0
        want = x.clone()
        for b, L_ in enumerate(Lb):
            row = want[b, c0:c0 + Cc]
            if mode == L.TAIL_REFLECT:
                for j in range(min(n, T - L_)):
                    row[:, L_ + j] = x[b, c0:c0 + Cc, abs(L_ - 2 - j)]
            elif mode == L.TAIL_REPLICATE and L_ % 2 == 1 and L_ < T:
                row[:, L_] = x[b, c0:c0 + Cc, L_ - 1]
            elif mode == L.TAIL_ZERO:
                row[:, L_:] = 0
        assert torch.equal(from_a4(xa), want), mode


# ------------------------------------------------------------------ Inferencer and CLI
def _inferencer(cfg):
    from adaptive_voice_conversion_b200.inference import Inferencer
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    return inf


def test_inference_padded(precision, monkeypatch):
    cfg = orc.default_config(80)
    inf = _inferencer(cfg)
    g = torch.Generator().manual_seed(11)
    src = torch.randint(100, 301, (40,), generator=g).tolist() + [17, 129]
    ref = torch.randint(100, 301, (40,), generator=g).tolist() + [9, 600]
    xs = [torch.randn((t, 80), generator=g).cuda() for t in src]
    cs = [torch.randn((t, 80), generator=g).cuda() for t in ref]
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    got = inf.inference_padded(xs, cs, batch_max=16)       # several batches, a padded batch size in the last
    assert inf.padded_captures > 0
    want = inf.inference_ragged(xs, cs)
    for i in range(len(xs)):
        assert got[i].shape == want[i].shape
        assert relerr(got[i], want[i]) < tol(precision, TOL_FP32, TOL_TF32), i
    # one batch of 64; a second call with different lengths on the same shape replays only
    inf.inference_padded(xs, cs)
    caps = inf.padded_captures
    src2 = [t - 3 if t > 20 else t for t in src]
    xs2 = [x[:t] for x, t in zip(xs, src2)]
    from adaptive_voice_conversion_b200.inference import padded_batches
    assert [b[1:] for b in padded_batches(src2, ref)] == [b[1:] for b in padded_batches(src, ref)]
    got2 = inf.inference_padded(xs2, cs)
    assert inf.padded_captures == caps
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    eager = inf.inference_padded(xs2, cs)
    for a, b in zip(got2, eager):
        assert torch.equal(a, b)


def test_pairs_cli_against_single_pair(tmp_path):
    cfg = orc.default_config(80)
    import yaml
    cfg_path = tmp_path / "config.yaml"
    cfg_path.write_text(yaml.safe_dump(cfg))
    from adaptive_voice_conversion_b200.model import AE
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0))
    torch.save(m.state_dict(), tmp_path / "model.ckpt")
    from scipy.io.wavfile import read, write
    rng, wavs = np.random.default_rng(0), []
    for i, secs in enumerate((0.6, 1.3, 2.1, 0.9)):
        t = np.arange(int(secs * 24000)) / 24000
        y = 0.3 * np.sin(2 * np.pi * (120 + 40 * i) * t * (1 + 0.2 * t)) + 0.02 * rng.standard_normal(t.size)
        wavs.append(str(tmp_path / f"w{i}.wav"))
        write(wavs[-1], 24000, (y * 32767).astype(np.int16))
    pairs = [(0, 1), (2, 3), (3, 0), (1, 2)]
    lines = [f"{wavs[a]} {wavs[b]} o{k}.npy" for k, (a, b) in enumerate(pairs)]
    lines += [f"{wavs[a]} {wavs[b]} o{k}" for k, (a, b) in enumerate(pairs)]
    pf = tmp_path / "pairs.txt"
    pf.write_text("\n".join(lines) + "\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", str(cfg_path), "-m", str(tmp_path / "model.ckpt"),
            "-gl_iters", "8"]
    out = tmp_path / "out"
    subprocess.run(base + ["-pairs", str(pf), "-o", str(out)], check=True, env=env, cwd=str(tmp_path))
    for k, (a, b) in enumerate(pairs):
        single = tmp_path / f"s{k}.npy"
        subprocess.run(base + ["-s", wavs[a], "-t", wavs[b], "-o", str(single)], check=True, env=env, cwd=str(tmp_path))
        got, want = np.load(out / f"o{k}.npy"), np.load(single)
        assert got.shape == want.shape
        assert relerr(torch.from_numpy(got), torch.from_numpy(want)) < TOL_TF32, k
        rate, y = read(out / f"o{k}.wav")
        assert rate == 24000 and y.size > 0
