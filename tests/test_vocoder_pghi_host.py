"""CPU: the PGHI start phase -- the phase-derivative formulas of tests/_pghi_ref.py on oracle STFTs of a sinusoid and
a click, the heap integration on hand-worked frames, the scan restatement against the heap on random and tied frames,
the argument checks of avc_pghi and avc_griffin_lim_from, the unchanged descriptor layout, and the -gl_init plumbing
of root inference.py."""
import ctypes as C
import os
import runpy
import subprocess
import sys

import numpy as np
import pytest

import oracle.audio_oracle as ao
import _pghi_ref as ref
from conftest import ROOT
from test_vocoder_fgla_host import FAKE, FakeInferencer, FakeVocoder, desc
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import vocoder as V

N, HOP = ao.N_FFT, ao.HOP


# ------------------------------------------------------------------ the phase-derivative formulas
def cosine(bin_, n=24000, phase=0.3):
    w0 = 2 * np.pi * bin_ / N
    return w0, np.cos(w0 * np.arange(n) + phase)


def trapezoid_error(bin_, bins, frames=np.arange(10, 70)):
    """max over frames of |wrapped (trapezoid of dt at f-1 and f) - (the STFT's own phase advance)| per bin."""
    w0, y = cosine(bin_)
    X = ao.stft(y)
    dt, _, _ = ref.derivatives(np.abs(X))
    out = {}
    for k in bins:
        est = 0.5 * (dt[frames - 1, k] + dt[frames, k])
        true = np.angle(X[frames, k] / X[frames - 1, k])
        out[k] = float(np.abs(ref.wrap(est - true)).max())
        assert np.abs(ref.wrap(w0 * HOP - true)).max() < 1e-5   # the sinusoid advances by w0 hop per frame
    return out


def test_sinusoid_on_its_bin_advances_by_w0_hop():
    """Centred on bin 100, the slope term vanishes by symmetry up to the negative-frequency image: the estimate is
    w0 hop (measured: 3.7e-7 rad)."""
    err = trapezoid_error(100.0, [100])
    assert err[100] < 1e-5, err


def test_sinusoid_off_bin_advance_is_close():
    """A cosine at bin 100.37: the Gaussian approximation of the Hann window leaves 0.010-0.083 rad at bins 99-102
    over frames 10-69 (measured on the oracle, phase offset 0.3).  Bound 0.1 rad."""
    err = trapezoid_error(100.37, [99, 100, 101, 102])
    assert max(err.values()) < 0.1, err


def click_steps(d, f=40):
    """(estimated dk, true per-bin phase step) at frame f for a click d samples after its centre."""
    y = np.zeros(24000)
    y[f * HOP + d] = 1.0
    X = ao.stft(y)
    _, dk, _ = ref.derivatives(np.abs(X))
    return dk[f], np.angle(X[f, 1:] / X[f, :-1])


def test_click_at_the_frame_centre_steps_by_minus_pi():
    """Frames f-1 and f+1 see the click symmetrically, so d_f l = 0 and the step is exactly -pi, as is the true
    step -2 pi (t0 - x + N/2) / N."""
    dk, true = click_steps(0)
    assert np.abs(dk + np.pi).max() < 1e-12
    assert np.abs(ref.wrap(true + np.pi)).max() < 1e-12


@pytest.mark.parametrize("d", [-137, 137, 60])
def test_click_off_centre_steps(d):
    """137 samples off the centre (frames f-1 and f+1 at 437 and -163 samples, inside the window's main support): the
    estimate is within 0.054 rad of -pi - 2 pi d / N (measured), bound 0.06.  Further out, where a neighbouring
    frame's window is nearly zero, the Gaussian approximation fails and nothing is claimed."""
    dk, true = click_steps(d)
    exact = -np.pi - 2 * np.pi * d / N
    assert np.abs(ref.wrap(true - exact)).max() < 1e-9
    assert np.abs(ref.wrap(dk - exact)).max() < 0.06
    assert np.abs(ref.wrap(0.5 * (dk[1:] + dk[:-1]) - true)).max() < 0.06


def test_significance_and_silence():
    S = np.array([[0.0, 1e-7, 1.0, 2.0], [3.0, 0.0, 1e-4, 5.0]])
    _, _, sig = ref.derivatives(S, tol=1e-5)
    assert sig.tolist() == [[False, False, True, True], [True, False, True, True]]
    _, _, sig = ref.derivatives(np.zeros((3, 5)))
    assert not sig.any()
    phi, par = ref.pghi_heap(np.zeros((3, 5)))
    assert not phi.any() and not par.any()


# ------------------------------------------------------------------ the heap integration, by hand
def test_heap_one_frame_by_hand():
    """No previous frame: the largest bin (k=4, an island of its own) is seeded first, then the largest of the rest
    (k=1), which reaches k=0 and k=2; k=3 is insignificant."""
    s = np.array([1.0, 3.0, 2.0, 0.0, 5.0])
    dk = np.array([0.1, 0.2, 0.4, 0.8, 1.6])
    par, phi = ref.heap_frame(np.zeros(5), np.zeros(5, bool), s, s > 0, dk_cur=dk)
    assert par.tolist() == [ref.RIGHT, ref.SEED, ref.LEFT, ref.NONE, ref.SEED]
    np.testing.assert_array_equal(phi, [-0.5 * (0.2 + 0.1), 0.0, 0.5 * (0.2 + 0.4), 0.0, 0.0])


def test_heap_two_frames_by_hand():
    """Sources (f-1, 0) = 4 and (f-1, 2) = 1.  (f-1, 0) assigns (f, 0).  Then (f-1, 2) and (f, 0) tie at 1 and the
    frame f-1 entry pops first, so (f, 2) comes in time and reaches (f, 1) before (f, 0) pops: k=1 is right-parented.
    k=4 has no source and is seeded."""
    sp = np.array([4.0, 0.0, 1.0, 0.0, 0.0])
    sc = np.array([1.0, 3.0, 2.0, 0.0, 5.0])
    phi_prev = np.array([0.3, 0.0, -1.0, 0.0, 0.0])
    dt_prev = np.array([1.0, 9.0, 2.0, 9.0, 9.0])
    dt_cur = np.array([3.0, 9.0, 4.0, 9.0, 9.0])
    dk = np.array([0.1, 0.2, 0.4, 0.8, 1.6])
    par, phi = ref.heap_frame(sp, sp > 0, sc, sc > 0, phi_prev, dt_prev, dt_cur, dk)
    assert par.tolist() == [ref.TIME, ref.RIGHT, ref.TIME, ref.NONE, ref.SEED]
    phi2 = -1.0 + 0.5 * (2.0 + 4.0)
    np.testing.assert_array_equal(phi, [0.3 + 0.5 * (1.0 + 3.0), phi2 - 0.5 * (0.4 + 0.2), phi2, 0.0, 0.0])
    # the same frames through the scan restatement
    par_s, phi_s = ref.scan_frame(sp, sp > 0, sc, sc > 0, phi_prev, dt_prev, dt_cur, dk)
    assert par_s.tolist() == par.tolist()
    np.testing.assert_allclose(phi_s, phi, rtol=0, atol=1e-15)


# ------------------------------------------------------------------ the scan restatement against the heap
def random_frames(rng, B, K, levels=None):
    """B frame pairs of K bins: uniform magnitudes, or quantised to `levels` values (heavy ties); random
    insignificant bins; a fifth of the pairs without any significant previous bin and some all-silent frames."""
    if levels:
        s = rng.integers(1, levels + 1, (2, B, K)).astype(np.float64)
    else:
        s = rng.uniform(0.05, 1.0, (2, B, K))
    sig = rng.uniform(size=(2, B, K)) > rng.uniform(0.0, 0.6, (2, B, 1))
    sig[0, rng.uniform(size=B) < 0.2] = False
    sig[1, rng.uniform(size=B) < 0.05] = False
    return s[0], sig[0], s[1], sig[1]


@pytest.mark.parametrize("levels", [None, 2, 3])
def test_scan_parents_equal_the_heap_on_random_frames(levels):
    rng = np.random.default_rng(7 + (levels or 0))
    n = 0
    for K in range(1, 24):
        sp, sigp, sc, sigc = random_frames(rng, 150, K, levels)
        par = ref.scan_parents(*ref.keys(sp, sigp, sc, sigc))
        for b in range(len(sp)):
            want, _ = ref.heap_frame(sp[b], sigp[b], sc[b], sigc[b])
            assert par[b].tolist() == want.tolist(), (K, sp[b], sigp[b], sc[b], sigc[b])
            n += 1
    assert n == 23 * 150


def test_scan_integration_equals_the_heap_on_utterances():
    rng = np.random.default_rng(3)
    for S in (np.abs(rng.standard_normal((30, 64))) ** 3,                       # wide dynamic range
              np.round(rng.uniform(0, 3, (20, 48))),                            # three levels and zeros
              np.abs(ao.stft(rng.standard_normal(3000)))[:, :200]):
        S[S < 0.01 * S.max()] *= rng.uniform(0, 1) < 0.5
        phi_h, par_h = ref.pghi_heap(S)
        phi_s, par_s = ref.pghi_scan(S)
        np.testing.assert_array_equal(par_s, par_h)
        assert np.abs(ref.wrap(phi_s - phi_h)).max() < 1e-9
        assert set(np.unique(par_h)) >= {ref.TIME, ref.LEFT, ref.RIGHT, ref.SEED}


# ------------------------------------------------------------------ the C entry points
def test_pghi_arguments_are_rejected_before_a_launch():
    lib = L.load()
    cases = [({}, 0.0, "tol"), ({}, 1.0, "tol"), ({}, -1e-5, "tol"), ({}, 2.0, "tol"), ({}, float("nan"), "tol"),
             ({}, float("inf"), "tol"), ({}, float("-inf"), "tol"),
             ({"mag": None}, 1e-5, "null mag or X"), ({"X": None}, 1e-5, "null mag or X"),
             ({"segs": None}, 1e-5, "utterance table"), ({"n_seg": 0}, 1e-5, "utterance table")]
    n0 = L.launch_count()
    for patch, tol, msg in cases:
        rc = lib.avc_pghi(C.byref(desc(**patch)), tol, C.c_void_p(FAKE), None)
        assert rc == L.ERR_INVALID, (patch, tol)
        assert msg in L.last_error(), (patch, L.last_error())
    rc = lib.avc_pghi(C.byref(desc(n_fft=1024)), 1e-5, None, None)
    assert rc == L.ERR_UNSUPPORTED and "n_fft" in L.last_error()
    assert L.launch_count() == n0


def test_griffin_lim_start_is_checked_before_a_launch():
    """avc_griffin_lim_from checks its start, the PGHI tolerance and every check of avc_griffin_lim before its first
    launch, so a bad momentum with the PGHI start enqueues nothing either."""
    lib = L.load()
    n0 = L.launch_count()
    for v in (3, -1, 7):
        rc = lib.avc_griffin_lim_from(C.byref(desc(momentum=0.0)), v, 1e-5, None)
        assert rc == L.ERR_INVALID and "unknown start" in L.last_error()
    for tol in (0.0, 1.0, -1e-5, float("nan"), float("inf")):
        rc = lib.avc_griffin_lim_from(C.byref(desc(momentum=0.0)), L.GL_START_PGHI, tol, None)
        assert rc == L.ERR_INVALID and "tol" in L.last_error(), tol
    for start in (L.GL_START_ZERO, L.GL_START_X, L.GL_START_PGHI):
        for patch, msg in (({"momentum": 1.0}, "momentum"), ({"momentum": float("nan")}, "momentum"),
                           ({"momentum": 0.5, "X_prev": None}, "needs X_prev"),
                           ({"momentum": 0.5, "X_prev": FAKE + 8}, "overlaps X"),
                           ({"X": None}, "null mag, X"), ({"mag": None}, "null mag, X"), ({"n_iter": -1}, "n_iter")):
            rc = lib.avc_griffin_lim_from(C.byref(desc(**patch)), start, 1e-5, None)
            assert rc == L.ERR_INVALID and msg in L.last_error(), (start, patch, L.last_error())
    assert L.launch_count() == n0


def test_descriptor_layout_and_its_mirror(tmp_path):
    """Every field of the header's avc_audio_desc sits at the ctypes mirror's offset, the old fields where they were
    (momentum 44, segs 48, mag_db 96, X_prev 104), and the size is unchanged: the start is an argument of
    avc_griffin_lim_from, which the header explains."""
    fields = [f for f, _ in L.AudioDesc._fields_]
    prog = ('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(){'
            + "".join(f'printf("%zu\\n", offsetof(avc_audio_desc, {f}));' for f in fields)
            + 'printf("%zu\\n", sizeof(avc_audio_desc));return 0;}\n')
    (tmp_path / "o.c").write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "o.c"), "-o", str(tmp_path / "o")])
    got = [int(v) for v in subprocess.check_output([str(tmp_path / "o")]).split()]
    assert got == [getattr(L.AudioDesc, f).offset for f in fields] + [C.sizeof(L.AudioDesc)]
    at = dict(zip(fields + ["sizeof"], got))
    assert [at[f] for f in ("momentum", "segs", "mag_db", "X_prev", "sizeof")] == [44, 48, 96, 104, 112]
    hdr = open(os.path.join(ROOT, "include", "avc_b200.h")).read()
    for name in ("ZERO", "X", "PGHI"):
        assert f"#define AVC_GL_START_{name} {getattr(L, 'GL_START_' + name)}" in hdr


def test_parent_codes_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "avc_b200.h")).read()
    for name in ("NONE", "TIME", "LEFT", "RIGHT", "SEED"):
        assert f"#define AVC_PGHI_{name} {getattr(L, 'PGHI_' + name)}" in hdr
        assert getattr(L, "PGHI_" + name) == getattr(ref, name)


# ------------------------------------------------------------------ Python and CLI
def test_params_default_to_zero_phase():
    hp = V.AudioParams()
    assert hp.gl_init == "zero" and hp.pghi_tol == ref.TOL


def test_bad_init_is_refused_before_any_work():
    with pytest.raises(ValueError, match="init"):
        V._init("random", V.AudioParams())
    with pytest.raises(ValueError, match="init"):
        V._init(None, V.AudioParams(gl_init="pghi "))
    assert V._init(None, V.AudioParams(gl_init="pghi")) == "pghi"


@pytest.mark.parametrize("flags,expect", [([], "zero"), (["-gl_init", "pghi"], "pghi"), (["-gl_init", "zero"], "zero")])
def test_cli_gl_init_reaches_the_vocoder(tmp_path, monkeypatch, flags, expect):
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
    assert voc.hp == V.AudioParams(gl_init=expect)


class PairsVocoder(FakeVocoder):
    def mel_to_wav(self, mels):
        import torch
        self.synthesised = len(mels)
        return [torch.zeros(8) for _ in mels]


class PairsInferencer(FakeInferencer):
    attr = None

    def __init__(self, config, args, vocoder=None):
        self.vocoder = vocoder

    def inference_padded(self, srcs, tgts):
        return [s.clone() for s in srcs]

    def write_wav_to_file(self, wav, path):
        open(path, "wb").close()


@pytest.mark.parametrize("flags,expect", [([], "zero"), (["-gl_init", "pghi"], "pghi")])
def test_cli_pairs_gl_init_reaches_the_vocoder(tmp_path, monkeypatch, flags, expect):
    import torch
    import adaptive_voice_conversion_b200.inference as I
    import adaptive_voice_conversion_b200.utils as U
    monkeypatch.setattr(I, "Inferencer", PairsInferencer)
    monkeypatch.setattr(U, "local_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(V, "Vocoder", PairsVocoder)
    for name in ("a", "b"):
        np.save(tmp_path / f"{name}.npy", np.ones((256, 512), np.float32))
    (tmp_path / "pairs.txt").write_text(f"{tmp_path / 'a.npy'} {tmp_path / 'b.npy'} out.wav\n")
    monkeypatch.setattr(sys, "argv", ["inference.py", "-c", os.path.join(ROOT, "config.yaml"),
                                      "-pairs", str(tmp_path / "pairs.txt"), "-o", str(tmp_path / "out"), *flags])
    FakeVocoder.made.clear()
    with pytest.raises(SystemExit) as e:
        runpy.run_path(os.path.join(ROOT, "inference.py"), run_name="__main__")
    assert e.value.code == 0
    voc, = FakeVocoder.made
    assert voc.hp == V.AudioParams(gl_init=expect) and voc.synthesised == 1
    assert (tmp_path / "out" / "out.wav").exists()


def test_cli_refuses_an_unknown_init(tmp_path, monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["inference.py", "-c", os.path.join(ROOT, "config.yaml"), "-s", "s.npy", "-t",
                                      "t.npy", "-o", "o.wav", "-gl_init", "random"])
    with pytest.raises(SystemExit):
        runpy.run_path(os.path.join(ROOT, "inference.py"), run_name="__main__")
    assert "gl_init" in capsys.readouterr().err
