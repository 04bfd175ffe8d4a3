"""CPU: fast Griffin-Lim (momentum) -- the argument checks of the C entry points, the float64 momentum loop
(tests/_fgla_ref.py) against the plain oracle loop and a two-iteration example written out here, and the -gl_iters /
-gl_momentum plumbing of root inference.py."""
import ctypes as C
import os
import runpy
import subprocess
import sys

import numpy as np
import pytest

import oracle.audio_oracle as ao
import _fgla_ref as ref
from conftest import ROOT
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import vocoder as V

FAKE = 1 << 24            # never dereferenced: every case fails validation before a launch
N_FRAMES = 10
X_BYTES = N_FRAMES * 1025 * 8
assert FAKE > X_BYTES     # so that X_prev below X is still an address


def desc(**kw):
    d = L.AudioDesc(n_fft=2048, hop=300, win=1200, n_seg=1, n_frames=N_FRAMES, n_samples=300 * (N_FRAMES - 1),
                    n_iter=4, mode=L.STFT_PROJECT, segs=FAKE, y=FAKE, mag=FAKE, X=FAKE, frames=FAKE,
                    X_prev=FAKE + X_BYTES)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("fn", ["avc_griffin_lim", "avc_stft"])
def test_momentum_arguments_are_rejected_before_a_launch(fn):
    lib = L.load()
    cases = [({"momentum": -0.1}, "momentum"), ({"momentum": 1.0}, "momentum"), ({"momentum": 1.5}, "momentum"),
             ({"momentum": float("nan")}, "momentum"), ({"momentum": float("inf")}, "momentum"),
             ({"momentum": float("-inf")}, "momentum"),
             ({"momentum": 0.99, "X_prev": None}, "needs X_prev"),
             ({"momentum": 0.5, "X_prev": FAKE}, "overlaps X"),
             ({"momentum": 0.5, "X_prev": FAKE + 8}, "overlaps X"),
             ({"momentum": 0.5, "X_prev": FAKE + X_BYTES - 8}, "overlaps X"),
             ({"momentum": 0.5, "X_prev": FAKE - X_BYTES + 8}, "overlaps X")]
    if fn == "avc_stft":
        cases += [({"mode": L.STFT_PROJECT_FIRST, **patch}, msg) for patch, msg in cases]
    n0 = L.launch_count()
    for patch, msg in cases:
        rc = getattr(lib, fn)(C.byref(desc(**patch)), None)
        assert rc == L.ERR_INVALID, patch
        assert msg in L.last_error(), (patch, L.last_error())
    assert L.launch_count() == n0


def test_struct_keeps_the_offsets_of_the_old_fields(tmp_path):
    """momentum takes the old int32 `reserved` slot (offset 44) and X_prev is appended: no old field moves."""
    fields = ["momentum", "segs", "mag_db", "X_prev"]
    prog = ('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", '
            + ", ".join(f"offsetof(avc_audio_desc, {f})" for f in fields) + ', sizeof(avc_audio_desc));return 0;}\n')
    (tmp_path / "o.c").write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "o.c"), "-o", str(tmp_path / "o")])
    got = [int(v) for v in subprocess.check_output([str(tmp_path / "o")]).split()]
    assert got == [getattr(L.AudioDesc, f).offset for f in fields] + [C.sizeof(L.AudioDesc)]
    assert got[:3] == [44, 48, 96] and got[3] == got[4] - 8 == 104


def spectrogram(n=3000, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 24000
    y = np.sin(2 * np.pi * 180 * t + 0.3 * np.sin(2 * np.pi * 5 * t)) + 0.05 * rng.standard_normal(n)
    return np.abs(ao.stft(y)) * rng.uniform(0.8, 1.2, (1 + n // 300, 1025))


def test_reference_without_momentum_is_the_plain_oracle_loop():
    S = spectrogram()
    X = S.astype(np.complex128)
    for _ in range(3):
        X = ao.griffin_lim_iteration(X, S)
    old = ao.istft(X)
    assert np.array_equal(ao.griffin_lim(S, 3), old)
    assert np.array_equal(ref.griffin_lim(S, 3), old)
    assert np.array_equal(ref.griffin_lim(S, 3, momentum=0.0), old)


def test_reference_momentum_one_iteration_is_plain_and_two_follow_the_definition():
    S = spectrogram(seed=1)
    m = 0.99
    assert np.array_equal(ref.griffin_lim(S, 1, momentum=m), ao.griffin_lim(S, 1))
    c = m / (1 + m)
    E1 = ao.stft(ao.istft(S))
    X1 = S * E1 / np.maximum(1e-8, np.abs(E1))
    E2 = ao.stft(ao.istft(X1))
    A2 = E2 - c * E1
    X2 = S * A2 / np.maximum(1e-8, np.abs(A2))
    two = ao.istft(X2)
    assert np.array_equal(ref.griffin_lim(S, 2, momentum=m), two)
    assert not np.allclose(two, ao.griffin_lim(S, 2))


def test_params_default_to_plain_griffin_lim():
    assert V.AudioParams().momentum == 0.0


class FakeVocoder:
    made = []

    def __init__(self, n_mels=None, hp=None, device=None):
        self.n_mels, self.hp = n_mels, hp
        FakeVocoder.made.append(self)

    def mel_to_wav(self, mels):
        import torch
        return [torch.zeros(8) for _ in mels]


class FakeInferencer:
    def __init__(self, config, args, vocoder=None):
        self.vocoder, self.attr = vocoder, None

    def inference_one_utterance(self, x, x_cond):
        return np.zeros(8, np.float32), x.numpy()

    def write_wav_to_file(self, wav, path):
        self.written = path


@pytest.mark.parametrize("flags,expect", [([], (100, 0.0)), (["-gl_iters", "32", "-gl_momentum", "0.99"], (32, 0.99))])
def test_cli_griffin_lim_flags_reach_the_vocoder(tmp_path, monkeypatch, flags, expect):
    import torch
    import adaptive_voice_conversion_b200.inference as I
    import adaptive_voice_conversion_b200.utils as U
    monkeypatch.setattr(I, "Inferencer", FakeInferencer)
    monkeypatch.setattr(U, "local_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(V, "Vocoder", FakeVocoder)
    np.save(tmp_path / "s.npy", np.ones((10, 4), np.float32))
    np.save(tmp_path / "t.npy", np.ones((7, 4), np.float32))
    monkeypatch.setattr(sys, "argv", ["inference.py", "-c", os.path.join(ROOT, "config.yaml"), "-s",
                                      str(tmp_path / "s.npy"), "-t", str(tmp_path / "t.npy"),
                                      "-o", str(tmp_path / "o.wav"), *flags])
    FakeVocoder.made.clear()
    runpy.run_path(os.path.join(ROOT, "inference.py"), run_name="__main__")
    voc, = FakeVocoder.made
    assert (voc.hp.n_iter, voc.hp.momentum) == expect
    assert voc.hp == V.AudioParams(n_iter=expect[0], momentum=expect[1])
