"""CPU: the vocoder's host side -- its float64 tables against the oracle, wav reading, the C structs of the audio
ABI, the resources of the audio kernels in the built library, and the plumbing of root inference.py."""
import ctypes
import os
import re
import runpy
import subprocess
import sys
import tempfile
import types

import numpy as np
import pytest
from scipy.io import wavfile

import oracle.audio_oracle as ao
from conftest import ROOT
from adaptive_voice_conversion_b200 import vocoder as V

AUDIO_KERNELS = ("stft_kernel", "istft_frames_kernel", "ola_kernel", "frame_power_kernel", "deemphasis_kernel",
                 "mel_gemm_kernel")


def test_params_are_the_tacotron_defaults():
    hp = V.AudioParams()
    assert (hp.sr, hp.n_fft, hp.hop_length, hp.win_length, hp.n_mels, hp.n_iter) == (24000, 2048, 300, 1200, 512, 100)
    assert (hp.preemphasis, hp.max_db, hp.ref_db, hp.top_db, hp.out_top_db) == (0.97, 100.0, 20.0, 15.0, 60.0)
    assert hp.n_bins == 1025 and hp.min_samples == 1025 and hp.min_frames == 5


@pytest.mark.parametrize("n_mels", [80, 512])
def test_tables_match_the_oracle(n_mels):
    hp = V.AudioParams(n_mels=n_mels)
    fb = V.mel_filterbank(hp)
    ref = ao.mel_filterbank(24000, 2048, n_mels)
    assert np.abs(fb - ref).max() <= 1e-12 * ref.max()
    M, Mref = V.mel_to_linear_matrix(fb), ao.mel_to_linear_matrix(ref)
    assert np.abs(M - Mref).max() <= 1e-10 * np.abs(Mref).max()
    f = np.array([0.0, 60.0, 999.0, 1000.0, 6400.0, 12000.0])
    assert np.allclose(V.hz_to_mel(f), ao.hz_to_mel(f), rtol=1e-14, atol=1e-14)


def test_trim_bounds_match_the_oracle():
    rng = np.random.default_rng(0)
    for top_db in (15, 60):
        p = 10.0 ** rng.uniform(-12, 0, 50)
        assert V.trim_bounds(p, 50 * 512 - 100, top_db) == ao.trim_bounds(p, 50 * 512 - 100, top_db)


def test_load_wav_scales_mixes_and_resamples(tmp_path):
    x = (np.arange(-8, 8) * 4096).astype(np.int16)
    st = np.stack([x, -x // 2], axis=1)
    p = str(tmp_path / "a.wav")
    wavfile.write(p, 24000, st)
    y = V.load_wav(p, 24000)
    assert y.dtype == np.float32
    assert np.array_equal(y, ((x / 32768.0 + (-x // 2) / 32768.0) / 2).astype(np.float32))
    t = np.arange(16000) / 16000
    wavfile.write(p, 16000, np.sin(2 * np.pi * 200 * t).astype(np.float32))
    y = V.load_wav(p, 24000)
    assert len(y) == 24000
    ref = np.sin(2 * np.pi * 200 * np.arange(24000) / 24000)
    assert np.abs(y[1000:-1000] - ref[1000:-1000]).max() < 1e-3


def test_audio_structs_match_header_sizes():
    from adaptive_voice_conversion_b200 import _lib as L
    prog = ('#include <stdio.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu\\n", sizeof(avc_audio_seg), '
            'sizeof(avc_audio_desc), sizeof(avc_mel_desc));return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write(prog)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(L.AudioSeg), ctypes.sizeof(L.AudioDesc), ctypes.sizeof(L.MelDesc)]
    assert V._SEG.itemsize == sizes[0]


def test_audio_kernels_use_no_stack_or_local_memory():
    from adaptive_voice_conversion_b200 import _lib as L
    L.load()
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and "REG:" in line and any(k in fn for k in AUDIO_KERNELS):
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    found = {k for k in AUDIO_KERNELS if any(k in fn for fn in res)}
    assert found == set(AUDIO_KERNELS), sorted(res)
    for fn, r in res.items():
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (fn, r)


class FakeInferencer:
    """Records what root inference.py hands the Inferencer."""
    made = []

    def __init__(self, config, args, vocoder=None):
        self.config, self.args, self.vocoder = config, args, vocoder
        self.attr = None
        FakeInferencer.made.append(self)

    def inference_one_utterance(self, x, x_cond):
        self.got = (x.clone(), x_cond.clone())
        return None, (x[:, :3] * 2).numpy()

    def write_wav_to_file(self, wav, path):
        raise AssertionError("a .npy output must not write a wav")


def test_cli_npy_plumbing_is_unchanged(tmp_path, monkeypatch):
    import torch
    import adaptive_voice_conversion_b200.inference as I
    import adaptive_voice_conversion_b200.utils as U
    monkeypatch.setattr(I, "Inferencer", FakeInferencer)
    monkeypatch.setattr(U, "local_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(V, "Vocoder", lambda *a, **k: pytest.fail("no vocoder for .npy arguments"))
    src = np.arange(40, dtype=np.float64).reshape(10, 4)
    tgt = np.ones((7, 4), np.float32)
    np.save(tmp_path / "s.npy", src)
    np.save(tmp_path / "t.npy", tgt)
    out = tmp_path / "o.npy"
    monkeypatch.setattr(sys, "argv", ["inference.py", "-c", os.path.join(ROOT, "config.yaml"), "-s",
                                      str(tmp_path / "s.npy"), "-t", str(tmp_path / "t.npy"), "-o", str(out)])
    FakeInferencer.made.clear()
    runpy.run_path(os.path.join(ROOT, "inference.py"), run_name="__main__")
    inf, = FakeInferencer.made
    assert inf.vocoder is None
    x, c = inf.got
    assert x.dtype == torch.float32 and torch.equal(x, torch.from_numpy(src.astype(np.float32)))
    assert torch.equal(c, torch.from_numpy(tgt))
    assert np.array_equal(np.load(out), src.astype(np.float32)[:, :3] * 2)


class Float64AttrInferencer:
    """An Inferencer whose attr.pkl holds float64 statistics and whose conversions double the source."""
    made = []

    def __init__(self, config, args, vocoder=None):
        self.vocoder, self.model = vocoder, None
        self.attr = {"mean": np.array([0.1, -0.2, 0.3, 0.7]), "std": np.array([0.3, 1.1, 0.9, 2.5])}
        Float64AttrInferencer.made.append(self)

    def normalize(self, x):     # Inferencer's
        return (x - self.attr["mean"]) / self.attr["std"]

    def denormalize(self, x):
        return x * self.attr["std"] + self.attr["mean"]

    def inference_one_utterance(self, x, x_cond):
        self.got = x.clone()
        return None, (x * 2).numpy()

    def inference_with_codes(self, xs, codes):
        self.got = xs[0].clone()
        return [xs[0] * 2]


@pytest.mark.parametrize("target", [["-t", "t.npy"], ["-bank", "bank.pt", "-speaker", "p1"]])
def test_cli_single_mode_casts_float64_statistics(tmp_path, monkeypatch, target):
    """A float64 attr.pkl is cast to float32, as -pairs does: the model gets float32 mels and the .npy output is
    float32, normalised and denormalised on the device."""
    import torch
    import adaptive_voice_conversion_b200.inference as I
    import adaptive_voice_conversion_b200.speaker_bank as SB
    import adaptive_voice_conversion_b200.utils as U
    monkeypatch.setattr(I, "Inferencer", Float64AttrInferencer)
    monkeypatch.setattr(U, "local_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(SB.SpeakerBank, "load", staticmethod(lambda path, model: types.SimpleNamespace(
        code=lambda spec: torch.zeros(8))))
    src = np.random.default_rng(0).standard_normal((10, 4)).astype(np.float32)
    np.save(tmp_path / "s.npy", src)
    np.save(tmp_path / "t.npy", np.ones((7, 4), np.float32))
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "argv", ["inference.py", "-c", os.path.join(ROOT, "config.yaml"), "-a", "attr.pkl",
                                      "-s", "s.npy", *target, "-o", "o.npy"])
    Float64AttrInferencer.made.clear()
    runpy.run_path(os.path.join(ROOT, "inference.py"), run_name="__main__")
    inf, = Float64AttrInferencer.made
    mean, std = (torch.tensor([0.1, -0.2, 0.3, 0.7], dtype=torch.float32),
                 torch.tensor([0.3, 1.1, 0.9, 2.5], dtype=torch.float32))
    x = (torch.from_numpy(src) - mean) / std
    assert inf.got.dtype == torch.float32 and torch.equal(inf.got, x)
    out = np.load(tmp_path / "o.npy")
    assert out.dtype == np.float32 and np.array_equal(out, (x * 2 * std + mean).numpy())
