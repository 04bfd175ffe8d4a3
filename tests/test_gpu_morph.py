"""GPU: time-varying speaker morphs (AE.inference_morph).

* avc_morph_weights against float64 at every f and odd lengths; avc_norm_apply_morph against a float64 restatement over
  shuffle / no shuffle, SAME / UP residuals, K in {1, 2, 3, 64} and ragged lengths, nothing written past L_b, bad
  arguments rejected;
* contracts, fp32 and TF32, configs c80 / c512 / sn: one-hot weights constant over time equal inference_from_embeddings
  with that anchor bit for bit (every anchor index); zero-weight extra anchors and reordered batch companions change no
  bit; NaN or +-1e4 in the padding of x and of the weights change no bit; a constant mix agrees with the mixed code's
  conversion within rounding;
* a piecewise trajectory (A -> crossfade -> B, then a three-speaker mix) against the float64 decoder restatement of
  tests/_morph_ref.py (it mixes codes, the kernel mixes rows) on the engine's own latent;
* Inferencer.inference_morph: CUDA graph equal to eager, K differing within a batch, equal to the per-source calls;
* end to end: inference.py -bank -morph p301@0 equals -speaker p301 bit for bit; a multi-keyframe wav run writes a wav.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from _morph_ref import decoder_morph, layer_weights
from _sn_ref import sn_config
from adaptive_voice_conversion_b200 import _lib as L
from test_gpu_padded_inference import TOL_FP32, TOL_TF32, _inferencer, make_model, relerr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = {"c80": lambda: orc.default_config(80), "c512": lambda: orc.default_config(512), "sn": lambda: sn_config(80)}
SENTINEL = -7777.0


@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


def to_a4(x):
    B, Cc, T = x.shape
    return x.reshape(B, Cc // 4, 4, T).permute(0, 1, 3, 2).contiguous()


def from_a4(a):
    B, Cq, T, _ = a.shape
    return a.permute(0, 1, 3, 2).reshape(B, Cq * 4, T)


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ----------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("f", (1, 2, 4, 8))
def test_morph_weights_kernel(f):
    lib = L.load()
    g = torch.Generator().manual_seed(f)
    B, K, T = 6, 5, 203
    lens = torch.tensor([203, 1, 7, 9, 64, 121], dtype=torch.int32)
    w = torch.rand((B, K, T), generator=g) * (torch.rand((B, K, T), generator=g) > 0.3)
    w[:, 0] += 0.01                                                          # a positive sum everywhere
    for b in range(B):
        w[b, :, int(lens[b]):] = float("nan")                                 # never read
    T_l = 8 * -(-T // 8) // f + 3
    out = torch.full((B, T_l, K), SENTINEL, device="cuda")
    wd, ld = w.cuda(), lens.cuda()
    assert lib.avc_morph_weights(wd.data_ptr(), ld.data_ptr(), B, K, T, f, out.data_ptr(), T_l, 0) == 0
    torch.cuda.synchronize()
    for b in range(B):
        Lb = int(lens[b])
        ref = layer_weights(w[b], Lb, f).t()
        n = ref.shape[0]
        got = out[b].cpu().double()
        assert (got[:n] - ref).abs().max() < 4e-7, (b, f)
        assert (got[n:] == 0).all()
    for args in ((0, K, T, f, T_l), (B, 0, T, f, T_l), (B, L.MORPH_MAX_K + 1, T, f, T_l), (B, K, T, 3, T_l), (B, K, T, 16, T_l)):
        assert lib.avc_morph_weights(wd.data_ptr(), ld.data_ptr(), *args[:4], out.data_ptr(), args[4], 0) == L.ERR_INVALID


def morph_epilogue_ref(c, lens_c, shuffle, rows, wtab, res, res_mode, relu):
    """float64: c [B, Cout, Tout] raw conv, lens_c conv frames per sample, rows [B, K, 2 Cn], wtab [B, Tn, K]."""
    outs = []
    for b in range(c.shape[0]):
        Lc = int(lens_c[b])
        y = c[b:b + 1, :, :Lc].double()
        y = orc.pixel_shuffle_1d(y, 2) if shuffle else y
        y = orc.instance_norm(y)[0]
        Cn, Tn = y.shape
        wr = wtab[b, :Tn].double()                                            # [Tn, K]
        beta = wr @ rows[b, :, :Cn].double()
        gamma = wr @ rows[b, :, Cn:].double()
        y = y * gamma.t() + beta.t()
        if relu:
            y = torch.relu(y)
        if res is not None:
            r = res[b].double()
            y = y + (r[:, :Tn] if res_mode == L.RES_SAME else r[:, torch.arange(Tn) // 2])
        outs.append(y)
    return outs


@pytest.mark.parametrize("K", (1, 2, 3, 64))
@pytest.mark.parametrize("shuffle,res_mode", [(False, L.RES_NONE), (False, L.RES_SAME), (True, L.RES_UP), (True, L.RES_NONE)])
def test_norm_apply_morph_kernel(K, shuffle, res_mode):
    lib = L.load()
    g = torch.Generator().manual_seed(K * 7 + res_mode)
    B, Cout, Tout = 5, 64, 40
    Cn, Tn = (Cout // 2, 2 * Tout) if shuffle else (Cout, Tout)
    lens = torch.tensor([40, 1, 17, 33, 8], dtype=torch.int32)              # conv frames (len_div = len_mul = 1)
    c = torch.randn((B, Cout, Tout), generator=g) * 2 + 0.5
    rows = torch.randn((B, K, 2 * Cn), generator=g)
    w = torch.rand((B, Tn, K), generator=g)
    w = w / w.sum(2, keepdim=True)
    res = torch.randn((B, Cn, Tn if res_mode == L.RES_SAME else Tout), generator=g) if res_mode != L.RES_NONE else None
    for b in range(B):
        c[b, :, int(lens[b]):] = float("nan")
    ca, ra = to_a4(c).cuda(), rows.cuda()
    resa = to_a4(res).cuda() if res is not None else None
    out = torch.full((B, Cn // 4, Tn, 4), SENTINEL, device="cuda")
    wd, ld = w.cuda(), lens.cuda()
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups, d.Tin, d.Tout = B, 4, Cout, 1, 1, 1, Tout, Tout
    d.save_c, d.out, d.out_bstride = ca.data_ptr(), out.data_ptr(), Cn * Tn
    d.shuffle, d.norm, d.relu, d.eps = int(shuffle), 1, 1, 1e-5
    d.cond, d.cond_bstride = ra.data_ptr(), K * 2 * Cn
    if resa is not None:
        d.res, d.res_bstride, d.res_mode, d.res_T = resa.data_ptr(), resa[0].numel(), res_mode, resa.shape[2]
    assert lib.avc_norm_apply_morph(C.byref(d), ld.data_ptr(), 1, 1, wd.data_ptr(), K, 2 * Cn, 0) == 0
    torch.cuda.synchronize()
    got = from_a4(out.cpu())
    ref = morph_epilogue_ref(c, lens, shuffle, rows, w, res, res_mode, True)
    for b in range(B):
        n = ref[b].shape[1]
        err = float((got[b, :, :n].double() - ref[b]).abs().max() / (ref[b].abs().max() + 1e-30))
        assert err < 2e-6, (b, err)
        assert (got[b, :, n:] == SENTINEL).all()                            # nothing written past L_b
    # rejections
    for kk in (0, L.MORPH_MAX_K + 1):
        assert lib.avc_norm_apply_morph(C.byref(d), ld.data_ptr(), 1, 1, wd.data_ptr(), kk, 2 * Cn, 0) == L.ERR_INVALID
    assert lib.avc_norm_apply_morph(C.byref(d), ld.data_ptr(), 1, 1, None, K, 2 * Cn, 0) == L.ERR_INVALID
    assert lib.avc_norm_apply_morph(C.byref(d), None, 1, 1, wd.data_ptr(), K, 2 * Cn, 0) == L.ERR_INVALID
    d2 = L.ConvDesc.from_buffer_copy(d)
    d2.mask = out.data_ptr()
    assert lib.avc_norm_apply_morph(C.byref(d2), ld.data_ptr(), 1, 1, wd.data_ptr(), K, 2 * Cn, 0) == L.ERR_UNSUPPORTED
    d2 = L.ConvDesc.from_buffer_copy(d)
    d2.res, d2.res_mode, d2.res_bstride, d2.res_T = out.data_ptr(), L.RES_POOL, Cn * Tn, Tn
    assert lib.avc_norm_apply_morph(C.byref(d2), ld.data_ptr(), 2, 1, wd.data_ptr(), K, 2 * Cn, 0) == L.ERR_INVALID
    d2 = L.ConvDesc.from_buffer_copy(d)
    d2.cond = None
    assert lib.avc_norm_apply_morph(C.byref(d2), ld.data_ptr(), 1, 1, wd.data_ptr(), K, 2 * Cn, 0) == L.ERR_INVALID
    d2 = L.ConvDesc.from_buffer_copy(d)
    d2.Cout = 6
    assert lib.avc_norm_apply_morph(C.byref(d2), ld.data_ptr(), 1, 1, wd.data_ptr(), K, 2 * Cn, 0) == L.ERR_INVALID


# ----------------------------------------------------------------------------- contracts on the model
LENS = [203, 17, 128, 145]


def batch(cfg, K, seed=0, T=None):
    g = torch.Generator().manual_seed(seed)
    n_mels = cfg["SpeakerEncoder"]["c_in"]
    T = T or max(LENS)
    x = torch.randn((len(LENS), n_mels, T), generator=g)
    codes = torch.randn((len(LENS), K, cfg["SpeakerEncoder"]["c_out"]), generator=g)
    return x.cuda(), codes.cuda(), torch.tensor(LENS, dtype=torch.int32).cuda()


def random_weights(K, T, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand((len(LENS), K, T), generator=g)
    w[:, 0] += 0.05
    return w.cuda()


@pytest.mark.parametrize("cfg_name", list(CONFIGS))
def test_one_hot_weights_equal_inference_from_embeddings(precision, cfg_name):
    cfg = CONFIGS[cfg_name]()
    m = make_model(cfg)
    K = 3
    x, codes, lens = batch(cfg, K)
    T = x.shape[2]
    for j in range(K):
        w = torch.zeros(len(LENS), K, T, device="cuda")
        w[:, j] = 2.5                                                        # one-hot up to scale
        got = m.inference_morph(x, codes, w, lengths=lens)
        want = m.inference_from_embeddings(x, codes[:, j].contiguous(), lengths=lens)
        assert got.shape == want.shape and same_bits(got, want), (cfg_name, j)


@pytest.mark.parametrize("cfg_name", list(CONFIGS))
def test_invariances(precision, cfg_name):
    cfg = CONFIGS[cfg_name]()
    m = make_model(cfg)
    K = 2
    x, codes, lens = batch(cfg, K + 2, seed=3)
    T = x.shape[2]
    w = random_weights(K, T, 4)
    base = m.inference_morph(x, codes[:, :K].contiguous(), w, lengths=lens)
    # zero-weight extra anchors
    wz = torch.cat([w, torch.zeros(len(LENS), 2, T, device="cuda")], 1)
    assert same_bits(m.inference_morph(x, codes, wz, lengths=lens), base)
    wz2 = torch.cat([torch.zeros(len(LENS), 2, T, device="cuda"), w], 1)     # in front as well
    assert same_bits(m.inference_morph(x, torch.cat([codes[:, K:], codes[:, :K]], 1), wz2, lengths=lens), base)
    # reordered batch companions
    perm = torch.tensor([2, 0, 3, 1], device="cuda")
    got = m.inference_morph(x[perm], codes[perm, :K].contiguous(), w[perm], lengths=lens[perm])
    assert same_bits(got, base[perm])
    # padding of x and of the weights
    for fill in (float("nan"), 1e4, -1e4):
        xp, wp = x.clone(), w.clone()
        for b, n in enumerate(LENS):
            xp[b, :, n:] = fill
            wp[b, :, n:] = fill
        assert same_bits(m.inference_morph(xp, codes[:, :K].contiguous(), wp, lengths=lens), base), fill
    # dec is 0 past each sample's frames
    for b, n in enumerate(LENS):
        assert (base[b, :, 8 * -(-n // 8):] == 0).all()


@pytest.mark.parametrize("cfg_name", list(CONFIGS))
def test_constant_mix_matches_the_mixed_code(precision, cfg_name):
    cfg = CONFIGS[cfg_name]()
    m = make_model(cfg)
    x, codes, lens = batch(cfg, 3, seed=5)
    mix = torch.tensor([0.2, 0.5, 0.3], device="cuda")
    w = mix[None, :, None].expand(len(LENS), 3, x.shape[2]).contiguous()
    got = m.inference_morph(x, codes, w, lengths=lens)
    want = m.inference_from_embeddings(x, (mix[None, :, None] * codes).sum(1), lengths=lens)
    # rows of a mix and the row of the mixed code round differently (a few float32 ulps per AdaIN row).  In fp32 the
    # decoder carries that as a relative change of order 1e-6; in TF32 the first conv of every block rounds its output
    # to TF32, and an ulp can move such a rounding by one TF32 ulp (2^-11 relative), the padded path's own bound
    err = relerr(got, want)
    assert err < (1e-4 if precision == "fp32" else TOL_TF32), err


def test_lengths_none_and_validation(precision):
    cfg = orc.default_config(80)
    m = make_model(cfg)
    x, codes, lens = batch(cfg, 2, seed=6, T=150)
    w = random_weights(2, 150, 7)
    full = m.inference_morph(x, codes, w)
    assert same_bits(full, m.inference_morph(x, codes, w, lengths=torch.full((4,), 150, dtype=torch.int32)))
    n0 = L.launch_count()
    bad_w = w.clone()
    bad_w[1, :, 3] = 0
    for args, kw, msg in (((x, codes, bad_w), {}, "positive sum"),
                          ((x, codes, w.clone().fill_(-1)), {}, "positive sum"),
                          ((x, codes[:, :1], w), {}, "expected codes"),
                          ((x, codes.double(), w), {}, "float32"),
                          ((x, codes.cpu(), w), {}, "float32"),
                          ((x, torch.zeros(4, 65, 128, device="cuda"), torch.ones(4, 65, 150, device="cuda")), {}, "K=65"),
                          ((x, codes, w), {"lengths": torch.tensor([150, 3, 150, 150])}, "lengths must lie")):
        with pytest.raises(L.AvcError, match=msg):
            m.inference_morph(*args, **kw)
    assert L.launch_count() == n0
    # NaN past a sample's frames is not an error; a NaN on a valid frame is
    w2 = w.clone()
    w2[0, :, 100:] = float("nan")
    m.inference_morph(x, codes, w2, lengths=torch.tensor([100, 150, 150, 150]))
    with pytest.raises(L.AvcError, match="positive sum"):
        m.inference_morph(x, codes, w2, lengths=torch.tensor([101, 150, 150, 150]))


def trajectory(L_, T):
    """A -> crossfade -> B, then a three-speaker mix: [3, T] (frames past L_ hold garbage)."""
    w = torch.full((3, T), float("nan"))
    t = torch.arange(L_, dtype=torch.float64)
    a = ((t - 0.3 * L_) / (0.2 * L_)).clamp(0, 1)
    w[0, :L_] = (1 - a).float()
    w[1, :L_] = a.float()
    w[2, :L_] = 0
    tail = t >= 0.8 * L_
    w[:, :L_][:, tail] = torch.tensor([0.2, 0.3, 0.5])[:, None]
    return w


@pytest.mark.parametrize("cfg_name", ("c80", "c512"))
def test_trajectory_against_float64_restatement(precision, cfg_name):
    cfg = CONFIGS[cfg_name]()
    m = make_model(cfg)
    x, codes, lens = batch(cfg, 3, seed=8)
    T = x.shape[2]
    w = torch.stack([trajectory(n, T) for n in LENS]).cuda()
    dec = m.inference_morph(x, codes, w, lengths=lens)
    mu, lat = m.get_content_means(x, lengths=lens)                           # the engine's own latent
    P = {k: v for k, v in m.state_dict().items()}
    tf32 = precision == "tf32"
    for b, n in enumerate(LENS):
        z = mu[b:b + 1, :, :int(lat[b])]
        ref = decoder_morph(P, cfg, z, codes[b], w[b], n, tf32=tf32)
        got = dec[b:b + 1, :, :ref.shape[2]]
        err = relerr(got, ref)
        print(f"{cfg_name} {precision} sample {b} ({n} frames): max rel err {err:.2e}")
        assert err < (1e-5 if precision == "fp32" else 2e-3), (b, err)      # measured: 1.2e-6 and 5.2e-4 at most


def test_inferencer_graph_equals_eager(precision, monkeypatch):
    cfg = orc.default_config(80)
    inf = _inferencer(cfg)
    g = torch.Generator().manual_seed(12)
    lens = [150, 97, 203, 64, 130, 171]
    Ks = [1, 3, 2, 5, 1, 2]
    xs = [torch.randn((n, 80), generator=g).cuda() for n in lens]
    cs = [torch.randn((k, 128), generator=g).cuda() for k in Ks]
    ws = [torch.rand((k, n), generator=g).add_(0.01).cuda() for k, n in zip(Ks, lens)]
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    caps = inf.padded_captures
    got = inf.inference_morph(xs, cs, ws, batch_max=4)
    assert inf.padded_captures > caps
    again = inf.inference_morph(xs, cs, ws, batch_max=4)
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    eager = inf.inference_morph(xs, cs, ws, batch_max=4)
    for i, (a, b, c) in enumerate(zip(got, again, eager)):
        assert a.shape == (8 * -(-lens[i] // 8), 80)
        assert same_bits(a, b) and same_bits(a, c), i
    # each source alone, with its own K_i anchors and its own extent: the padded path's rounding bound
    for i in range(len(xs)):
        one = inf.model.inference_morph(xs[i].t()[None].contiguous(), cs[i][None], ws[i][None])
        assert relerr(one[0].t(), eager[i]) < (TOL_FP32 if precision == "fp32" else TOL_TF32), i


# ----------------------------------------------------------------------------- end to end
def test_morph_cli(tmp_path):
    from test_gpu_bank import write_train
    from test_gpu_fewshot import _checkpoint
    cfg = orc.default_config(80)
    cfg_path, ckpt = _checkpoint(tmp_path, cfg)
    write_train(tmp_path, 80)
    env = dict(os.environ, PYTHONPATH=ROOT)
    bank_path = str(tmp_path / "bank.pt")
    subprocess.run([sys.executable, os.path.join(ROOT, "speaker_bank.py"), "-c", cfg_path, "-m", ckpt, "-d", str(tmp_path),
                    "-set", "train", "-o", bank_path], check=True, env=env, cwd=str(tmp_path), capture_output=True)
    src = str(tmp_path / "s.npy")
    np.save(src, np.random.default_rng(2).standard_normal((173, 80)).astype(np.float32))
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", cfg_path, "-m", ckpt, "-bank", bank_path]
    subprocess.run(base + ["-s", src, "-speaker", "p301", "-o", str(tmp_path / "a.npy")], check=True, env=env, cwd=str(tmp_path))
    subprocess.run(base + ["-s", src, "-morph", "p301@0", "-o", str(tmp_path / "b.npy")], check=True, env=env, cwd=str(tmp_path))
    a, b = np.load(tmp_path / "a.npy"), np.load(tmp_path / "b.npy")
    assert a.shape == b.shape == (176, 80) and np.array_equal(a.view(np.int32), b.view(np.int32))
    # a wav source, several keyframes, a wav out
    from scipy.io.wavfile import read, write
    t = np.arange(int(1.5 * 24000)) / 24000
    y = 0.3 * np.sin(2 * np.pi * 140 * t * (1 + 0.2 * t)) + 0.02 * np.random.default_rng(3).standard_normal(t.size)
    write(str(tmp_path / "s.wav"), 24000, (y * 32767).astype(np.int16))
    subprocess.run(base + ["-s", str(tmp_path / "s.wav"), "-morph", "p300@0", "p300@0.4", "p302@0.6", "p301:0.5,p302:0.5@1.2",
                           "-o", str(tmp_path / "m.wav")], check=True, env=env, cwd=str(tmp_path))
    sr, out = read(str(tmp_path / "m.wav"))
    assert sr == 24000 and 0 < out.shape[0] <= (8 * -(-int(1.5 * 80 + 1) // 8) + 1) * 300
