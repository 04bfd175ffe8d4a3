"""CPU: the host side of padded batches of different-length utterances (AE.inference with lengths).

* every descriptor the padded path sends to avc_conv_block_tc gets a tensor-core plan, over padded extents of 17..600
  frames, at c_in 80 and 512 (the fake-library engine of tests/test_conv_tc2_plan.py);
* the slack invariant: at every reflect-padded conv, each sample of every length <= T has room for its reflected frames
  inside the layer's extent;
* the bucket grid of Inferencer.inference_padded is deterministic, covers every pair once and bounds the shape count;
* invalid lengths and pairs-file errors are rejected before any launch;
* the batch helpers the padded paths share: fill_rows, padded_batch, scatter_crops, exact_buckets and eval_mode.
"""
import os
import sys
import types

import pytest
import torch

import oracle.ae_oracle as orc
from test_conv_tc2_plan import cpu_engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


class VarlenRecorder:
    """Wraps the fake library of cpu_engine: records the varlen launches (kind, tensor extent, len_div, len_mul, n)."""

    def __init__(self, inner):
        self.inner, self.calls = inner, []

    def avc_varlen_tail(self, ptr, bstride, B, Cc, T, lens, div, mul, mode, n, stream):
        self.calls.append(("tail", T, div, mul, mode, n))
        return 0

    def avc_norm_apply_varlen(self, dref, lens, div, mul, stream):
        d = dref._obj
        self.calls.append(("norm", d.Tout, div, mul, int(d.res_mode) if d.res else 0, int(d.shuffle)))
        return 0

    def avc_time_mean_varlen_fwd(self, ptr, bstride, out, B, Cc, T, lens, div, mul, stream):
        self.calls.append(("mean", T, div, mul, 0, 0))
        return 0

    def __getattr__(self, name):
        return getattr(self.inner, name)


def padded_forward(e, P, B, T, Tc, c_in):
    from adaptive_voice_conversion_b200.engine import Lengths, varlen_extent
    lx, lc = Lengths(torch.full((B,), T, dtype=torch.int32)), Lengths(torch.full((B,), Tc, dtype=torch.int32))
    with torch.no_grad():
        emb, _ = e.speaker_fwd(P, torch.empty(B, c_in, varlen_extent(e.cfg, Tc, source=False)), False, lens=lc)
        mu4, ls4, ctx = e.content_fwd(P, torch.empty(B, c_in, varlen_extent(e.cfg, T, source=True)), False, lens=lx)
        dec4, _ = e.decoder_fwd(P, mu4, emb, False, lens=ctx["lens"])
    return dec4


@pytest.mark.parametrize("c_in", (80, 512))
def test_padded_descriptors_all_plan(monkeypatch, lib, c_in):
    """Padded extents of batches whose longest utterance has 17..600 frames (B = 1 and 64): no tensor-core rejection;
    every InstanceNorm block runs as a plain conv + avc_norm_apply_varlen."""
    e, P = cpu_engine(monkeypatch, lib, 132, c_in)
    rec = VarlenRecorder(e.lib)
    e.lib = rec
    step = 1 if c_in == 80 else 7
    for T in range(17, 601, step):
        for B in (1, 64) if T % 5 == 0 else (1,):
            rec.calls.clear()
            n_before = rec.inner.n
            dec4 = padded_forward(e, P, B, T, max(9, (T * 7) % 601), c_in)
            assert dec4.T == 8 * -(-dec4.T // 8)
            assert rec.inner.n > n_before and not rec.inner.rejected, (T, rec.inner.rejected[:3])
            norms = [c for c in rec.calls if c[0] == "norm"]
            # content: in_conv + 2 per block; decoder: in_conv + 2 per block
            ce, de = e.cfg["ContentEncoder"], e.cfg["Decoder"]
            assert len(norms) == 1 + 2 * ce["n_conv_blocks"] + 1 + 2 * de["n_conv_blocks"]
            assert sum(c[0] == "mean" for c in rec.calls) == 1
            assert [c[4] for c in rec.calls if c[0] == "tail"][-1] == 2     # the decoder output's zero tail is last


def test_slack_invariant_every_layer_every_length():
    """For every T up to 600 and every length 1..T, at every reflect-padded conv of both paths the sample's
    pad_right reflected frames lie inside the layer's extent, and the extent chain is conv_geometry's."""
    from adaptive_voice_conversion_b200.engine import Lengths, _varlen_layers, conv_geometry, varlen_extent
    for c_in in (80, 512):
        cfg = orc.default_config(c_in)
        for source in (True, False):
            layers = _varlen_layers(cfg, source)
            for T in range(1, 601):
                Te = varlen_extent(cfg, T, source)
                assert Te >= T and Te % 8 == 0
                # extent chain by conv_geometry == ceil arithmetic of Lengths
                c = cfg["ContentEncoder" if source else "SpeakerEncoder"]
                ext, div = Te, 1
                for s in c["subsample"][: c["n_conv_blocks"]]:
                    ext, div = conv_geometry(c["kernel_size"], s, ext)[2], div * s
                assert ext == Lengths(None, div).of(Te)
                lens = torch.arange(1, T + 1)
                for (div, mul), pr in layers:
                    ext = Lengths(None, div, mul).of(Te)
                    at = (lens + div - 1) // div * mul                 # every length 1..T at this layer
                    assert int(at.max()) + pr <= ext, (c_in, source, T, div, mul, pr)


def test_bucket_grid():
    from adaptive_voice_conversion_b200.inference import padded_batches, padded_extent
    g = torch.Generator().manual_seed(0)
    src = torch.randint(100, 601, (512,), generator=g).tolist()
    ref = torch.randint(100, 601, (512,), generator=g).tolist()
    a, b = padded_batches(src, ref, 64), padded_batches(list(src), list(ref), 64)
    assert a == b                                                   # deterministic
    seen = sorted(i for idx, *_ in a for i in idx)
    assert seen == list(range(512))                                 # every pair exactly once
    grid = {padded_extent(t) for t in range(100, 601)}
    assert len(grid) == 11
    for idx, T, Tc, B in a:
        assert len(idx) <= B <= 64 and B & (B - 1) == 0
        assert T in grid and Tc in grid
        assert all(src[i] <= T and ref[i] <= Tc for i in idx)
    assert len({(T, Tc, B) for _, T, Tc, B in a}) <= 8
    # any list: the shape count is bounded by the grid and the batch sizes, and small lists pad their batch size
    for n in (1, 3, 65, 200):
        p = padded_batches(src[:n], ref[:n], 64)
        assert sum(len(i) for i, *_ in p) == n
        assert all(B == min(64, 1 << (len(i) - 1).bit_length()) for i, _, _, B in p)
    assert padded_extent(17) == 32 and padded_extent(256) == 256 and padded_extent(257) == 320 and padded_extent(1025) == 1152
    with pytest.raises(ValueError):
        padded_batches([1, 2], [1], 4)


def test_batch_helpers():
    """fill_rows writes the rows in `rows` order (repeats included), keeps the tail and returns the lengths;
    padded_batch zero-fills with int32 lengths; scatter_crops crops to 8 ceil(T / 8); exact_buckets gives sorted keys
    with indices in input order; eval_mode restores the training mode and checks the status word on a normal exit only."""
    from adaptive_voice_conversion_b200.inference import fill_rows, padded_batch, scatter_crops
    from adaptive_voice_conversion_b200.utils import eval_mode, exact_buckets
    frames = [torch.full((3, n), float(k + 1)) for k, n in enumerate((5, 2, 7))]
    dst = torch.full((4, 3, 8), -1.0)
    assert fill_rows(dst, frames, [2, 0, 2, 1]) == [7, 5, 7, 2]
    for j, i in enumerate([2, 0, 2, 1]):
        n = frames[i].shape[1]
        assert torch.equal(dst[j, :, :n], frames[i]) and bool((dst[j, :, n:] == -1).all())
    x, lens = padded_batch(frames, [1, 2], 8, "cpu")
    assert x.shape == (2, 3, 8) and lens.dtype == torch.int32 and lens.tolist() == [2, 7]
    assert torch.equal(x[0, :, :2], frames[1]) and torch.equal(x[1, :, :7], frames[2])
    assert not x[0, :, 2:].any() and not x[1, :, 7:].any()
    out, dec = [None] * 3, torch.arange(2 * 3 * 24.0).view(2, 3, 24)
    scatter_crops(out, dec, [2, 0], [17, 9])
    assert out[1] is None and torch.equal(out[2], dec[0].t()) and torch.equal(out[0], dec[1, :, :16].t())
    assert exact_buckets([3, 1, 3, 1, 2], [1, 1, 1, 2, 1]) == [((1, 1), [1]), ((1, 2), [3]), ((2, 1), [4]), ((3, 1), [0, 2])]
    g = torch.Generator().manual_seed(0)
    src, ref = torch.randint(17, 25, (300,), generator=g).tolist(), torch.randint(9, 13, (300,), generator=g).tolist()
    b = exact_buckets(src, ref)
    assert [k for k, _ in b] == sorted({*zip(src, ref)}) and sorted(i for _, idx in b for i in idx) == list(range(300))
    assert all(idx == sorted(idx) and all((src[i], ref[i]) == k for i in idx) for k, idx in b)

    class Model(torch.nn.Module):
        checks = []

        def engine(self, dev):
            return types.SimpleNamespace(check_tc_status=lambda: self.checks.append(dev))
    m = Model()
    with eval_mode(m, "cuda:0"):
        assert not m.training
    assert m.training and m.checks == ["cuda:0"]
    with pytest.raises(RuntimeError, match="inside"):
        with eval_mode(m, "cuda:0"):
            raise RuntimeError("inside")
    assert m.training and m.checks == ["cuda:0"]
    m.eval()
    with eval_mode(m, "cuda:1"):
        pass
    assert not m.training and m.checks == ["cuda:0", "cuda:1"]


def test_invalid_lengths_rejected_before_any_launch(lib):
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200.model import _check_lengths
    x = torch.zeros(3, 80, 100)
    n0 = L.launch_count()
    ok = _check_lengths(torch.tensor([17, 100, 55]), x, 17, "t")
    assert ok.dtype == torch.int32 and ok.tolist() == [17, 100, 55]
    assert _check_lengths(None, x, 17, "t").tolist() == [100, 100, 100]
    bad = [torch.tensor([16, 100, 55]),            # below the minimum
           torch.tensor([17, 101, 55]),            # past the extent
           torch.tensor([17, 100]),                # batch-size mismatch
           torch.tensor([[17, 100, 55]]),          # wrong shape
           torch.tensor([17.0, 100.0, 55.0]),      # wrong dtype
           torch.tensor([True, True, True]),
           [17, 100, 55]]                          # not a tensor
    for v in bad:
        with pytest.raises(L.AvcError):
            _check_lengths(v, x, 17, "t")
    assert L.launch_count() == n0


def test_pairs_file_errors_name_the_line(tmp_path):
    sys.path.insert(0, ROOT)
    import inference as cli
    a = tmp_path / "a.npy"
    import numpy as np
    np.save(a, np.zeros((40, 80), np.float32))
    np.save(tmp_path / "short.npy", np.zeros((10, 80), np.float32))
    good = tmp_path / "good.txt"
    good.write_text(f"# comment\n{a} {a} out1.npy\n\n{a} {a}\n")
    pairs = cli.read_pairs(str(good))
    assert [(p[0], p[3]) for p in pairs] == [(2, "out1.npy"), (4, "a_to_a.wav")]
    for text, msg in ((f"{a}\n", "line 1"), (f"{a} {a}\n{a} {tmp_path / 'missing.npy'}\n", "line 2"),
                      (f"{a} {a} x y z\n", "line 1"), (f"{a} {a} out.txt\n", "line 1"), (f"{a} {a} sub/out.npy\n", "line 1")):
        f = tmp_path / "bad.txt"
        f.write_text(text)
        with pytest.raises(ValueError, match=msg):
            cli.read_pairs(str(f))
    with pytest.raises(ValueError, match="line 1"):
        cli.check_frames([(1, str(tmp_path / "short.npy"), str(a), "o.npy")], [10], [40], (17, 9))
    with pytest.raises(ValueError, match="line 3"):
        cli.check_frames([(3, str(a), str(tmp_path / "short.npy"), "o.npy")], [40], [8], (17, 9))
    cli.check_frames([(3, str(a), str(a), "o.npy")], [17], [9], (17, 9))
