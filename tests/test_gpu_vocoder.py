"""GPU: the vocoder kernels (csrc/audio.cu) against the float64 oracle (oracle/audio_oracle.py), their ragged-batch
and graph-replay determinism, their errors, and wav-to-wav conversion through inference.py and the Inferencer.

Inputs are seeded and synthetic (harmonic tones with vibrato, a noise burst, silence) at 24 kHz."""
import os
import pickle
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
import yaml
from scipy.io import wavfile

import oracle.ae_oracle as orc
import oracle.audio_oracle as ao
from conftest import ROOT

pytestmark = pytest.mark.gpu

SR = 24000


def utterance(n, seed, silence=(3000, 2500)):
    """Silence, a vibrato tone with 6 harmonics, a noise burst, more tone, silence; float32."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    f0 = rng.uniform(110, 220) * (1 + 0.03 * np.sin(2 * np.pi * rng.uniform(4, 6) * t))
    ph = 2 * np.pi * np.cumsum(f0) / SR
    y = sum(rng.uniform(0.05, 0.3) / k * np.sin(k * ph + rng.uniform(0, 6.3)) for k in range(1, 7))
    a, b = n // 3, n // 3 + n // 8
    y[a:b] += 0.2 * rng.standard_normal(b - a)
    y[:silence[0]] = 0
    y[n - silence[1]:] = 0
    return y.astype(np.float32)


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope="module")
def V():
    from adaptive_voice_conversion_b200 import vocoder
    return vocoder


LENGTHS = [1025, 1025 + 299, 4800, 24000 + 137]   # shortest legal, both reflect edges, multiple and not of hop


@pytest.mark.parametrize("preemph", [0.0, 0.97])
def test_stft_matches_oracle(V, preemph):
    ys = [utterance(n, i, silence=(0, 0)) for i, n in enumerate(LENGTHS)]
    got = V.stft([dev(y) for y in ys], preemphasis=preemph)
    mags = V.magnitude([dev(y) for y in ys], preemphasis=preemph)
    worst = 0.0
    for y, X, (mag, mag_db) in zip(ys, got, mags):
        yy = ao.preemphasis(y, preemph) if preemph else y.astype(np.float64)
        ref = ao.stft(yy)
        X = X.cpu().numpy()
        assert X.shape == ref.shape
        scale = np.abs(ref).max(axis=1, keepdims=True)
        err = (np.abs(X - ref) / scale).max()
        worst = max(worst, err)
        assert err < 1e-5, err
        assert (np.abs(mag.cpu().numpy() - np.abs(ref)) / scale).max() < 1e-5
        assert np.abs(mag_db.cpu().numpy() - ao.normalize_db(mag.cpu().numpy().astype(np.float64))).max() < 1e-6
    print(f"stft max error / frame max: {worst:.2e}")


def test_istft_matches_oracle(V):
    # an iSTFT needs 5 frames (its output must be long enough to be analysed again): 1200 samples at least
    ys = [utterance(n, 10 + i, silence=(0, 0)) for i, n in enumerate([1200, 1324, 4800, 24137])]
    specs = [ao.stft(y) for y in ys]
    got = V.istft([dev(s.astype(np.complex64)) for s in specs])
    got0 = V.istft([dev(np.abs(s).astype(np.float32)) for s in specs])      # zero-phase form (Griffin-Lim's start)
    for s, z, z0 in zip(specs, got, got0):
        ref, ref0 = ao.istft(s), ao.istft(np.abs(s))
        assert z.shape[0] == len(ref) == 300 * (s.shape[0] - 1)
        assert np.abs(z.cpu().numpy() - ref).max() < 1e-5 * np.abs(ref).max()
        # a zero-phase frame is a pulse at the frame's edges: the windowed part is a small difference of large terms,
        # so its error scale is the peak of the unwindowed inverse frames
        scale0 = np.abs(np.fft.irfft(np.abs(s), n=2048, axis=1)).max()
        assert np.abs(z0.cpu().numpy() - ref0).max() < 1e-5 * scale0


def test_one_griffin_lim_iteration_matches_oracle(V):
    rng = np.random.default_rng(5)
    S = [np.abs(ao.stft(utterance(n, 20 + i))) * rng.uniform(0.5, 1.5, (1 + n // 300, 1025)) for i, n in
         enumerate([6000, 9137])]
    got = V.griffin_lim([dev(s.astype(np.float32)) for s in S], n_iter=1)
    for s, z in zip(S, got):
        ref = ao.griffin_lim(s, 1)
        assert np.abs(z.cpu().numpy() - ref).max() < 1e-5 * np.abs(ref).max()


def test_griffin_lim_100_iterations_tracks_the_oracle(V):
    y = utterance(SR, 30)
    S = np.abs(ao.stft(y))
    z = V.griffin_lim([dev(S.astype(np.float32))])[0].cpu().numpy().astype(np.float64)
    ref = ao.griffin_lim(S, 100)
    rel = float(np.linalg.norm(z - ref) / np.linalg.norm(ref))
    sc, sc_ref = ao.spectral_convergence(S, z), ao.spectral_convergence(S, ref)
    print(f"griffin-lim 100 it: waveform rel L2 {rel:.3e}, spectral convergence {sc:.5f} (oracle {sc_ref:.5f})")
    assert rel < 1e-2, rel
    assert abs(sc - sc_ref) < 1e-3, (sc, sc_ref)


def denormalize(v):
    return 10.0 ** ((np.asarray(v, np.float64) * 100 - 100 + 20) / 20)


def compare_normalised(got, ref_lin):
    """got: normalised values from the device; ref_lin: the oracle's linear amplitudes.  Returns (max error in the
    normalised domain, the same over entries within 60 dB of their frame's peak, max amplitude error / frame peak).
    The normalised domain is 20 log10: an amplitude error d moves it by 0.087 d / a, so fp32's error of ~1e-7 of the
    frame peak reaches 1e-5 there only for entries more than ~60 dB below the peak."""
    ref = ao.normalize_db(ref_lin)
    peak = np.maximum(ref_lin.max(axis=1, keepdims=True), 1e-5)   # 1e-5: the amplitude floor of the dB step
    err = np.abs(got - ref)
    loud = ref_lin >= 1e-3 * peak
    amp = np.abs(denormalize(got) - denormalize(ref)) / peak
    return float(err.max()), float(err[loud].max()), float(amp.max())


@pytest.mark.parametrize("n_mels", [80, 512])
def test_get_spectrograms_matches_oracle(V, tmp_path, n_mels):
    voc = V.Vocoder(n_mels=n_mels)
    fb = ao.mel_filterbank(SR, 2048, n_mels)
    for i, n in enumerate([15000, 40000]):
        p = str(tmp_path / f"u{i}.wav")
        wavfile.write(p, SR, utterance(n, 40 + i))
        mel, mag = voc.get_spectrograms(p)
        y = V.load_wav(p, SR).astype(np.float64)
        rmel, rmag = ao.get_spectrograms(y, n_mels=n_mels)
        rmag_lin = np.abs(ao.stft(ao.preemphasis(ao.trim(y, 15))))
        assert mel.dtype == np.float32 and mag.dtype == np.float32
        assert mel.shape == rmel.shape and mag.shape == rmag.shape, (mel.shape, rmel.shape)
        em, em_loud, em_amp = compare_normalised(mel, rmag_lin @ fb.T)
        eg, eg_loud, eg_amp = compare_normalised(mag, rmag_lin)
        print(f"n_mels={n_mels} T={mel.shape[0]}: normalised max err mel {em:.2e} mag {eg:.2e}; within 60 dB of the "
              f"frame peak mel {em_loud:.2e} mag {eg_loud:.2e}; amplitude / frame peak mel {em_amp:.2e} mag {eg_amp:.2e}")
        assert em_loud < 1e-5 and eg_loud < 1e-5, (em_loud, eg_loud)
        assert em_amp < 1e-5 and eg_amp < 1e-5, (em_amp, eg_amp)


def test_melspectrogram2wav_stages_match_oracle(V):
    """Mel -> magnitude matches the oracle; 100 Griffin-Lim iterations on it converge as far as the oracle's (a mel's
    pseudo-inverse is no consistent spectrogram, so the iterations drift apart in phase: the spectral convergence is
    the comparable quantity, and fp32 may land within 1 % of it on either side); de-emphasis and trim of the device's Griffin-Lim output give what melspectrogram2wav returns."""
    voc = V.Vocoder(n_mels=80)
    mel = ao.get_spectrograms(utterance(12000, 50).astype(np.float64), n_mels=80)[0].astype(np.float32)
    S = voc.mel_to_mag([dev(mel)])[0]
    Sref = ao.mel_to_mag(mel)
    assert (np.abs(S.cpu().numpy() - Sref) / Sref.max(axis=1, keepdims=True)).max() < 1e-5
    gl = V.griffin_lim([S])[0].cpu().numpy().astype(np.float64)
    ref = ao.griffin_lim(Sref, 100)
    sc, sc_ref = ao.spectral_convergence(Sref, gl), ao.spectral_convergence(Sref, ref)
    rel = float(np.linalg.norm(gl - ref) / np.linalg.norm(ref))
    print(f"mel-derived griffin-lim 100 it: waveform rel L2 {rel:.3e}, spectral convergence {sc:.5f} "
          f"(oracle {sc_ref:.5f})")
    assert sc < 1.01 * sc_ref, (sc, sc_ref)
    wav = voc.melspectrogram2wav(mel)
    tail = ao.trim(ao.deemphasis(gl), 60)
    assert wav.dtype == np.float32 and np.isfinite(wav).all() and len(wav) == len(tail)
    assert np.abs(wav - tail).max() < 1e-5 * np.abs(tail).max()


def test_deemphasis_and_trim_on_device(V):
    ys = [utterance(n, 60 + i, silence=s) for i, (n, s) in enumerate([(5000, (0, 0)), (31001, (3000, 2500)),
                                                                         (1025, (0, 0))])]
    got = V.deemphasis([dev(y) for y in ys])
    for y, z in zip(ys, got):
        ref = ao.deemphasis(y)
        assert np.abs(z.cpu().numpy() - ref).max() < 1e-5 * np.abs(ref).max()
    for top_db in (15, 60):
        trimmed = V.trim([dev(y) for y in ys], top_db)
        for y, z in zip(ys, trimmed):
            s, e = ao.trim_bounds(ao.frame_power(y), len(y), top_db)
            assert torch.equal(z.cpu(), torch.from_numpy(y[s:e]))


def test_ragged_batches_are_bitwise_per_utterance(V):
    voc = V.Vocoder(n_mels=80)
    wavs = [dev(utterance(n, 70 + i)) for i, n in enumerate([9000, 15001, 9000, 20000])]
    batch = voc.wav_to_mel(wavs)
    for w, (mel, mag) in zip(wavs, batch):
        m1, g1 = voc.wav_to_mel([w])[0]
        assert torch.equal(mel, m1) and torch.equal(mag, g1)
    mels = [m for m, _ in batch]
    out = voc.mel_to_wav(mels, n_iter=10)
    again = voc.mel_to_wav(mels, n_iter=10)
    for m, a, b in zip(mels, out, again):
        assert torch.equal(a, b)
        assert torch.equal(a, voc.mel_to_wav([m], n_iter=10)[0])


def test_griffin_lim_graph_replay_is_bitwise(V):
    S = [dev(np.abs(ao.stft(utterance(n, 80 + i))).astype(np.float32)) for i, n in enumerate([7000, 12345])]
    plan = V.GriffinLim(S, n_iter=8)
    eager = [y.clone() for y in plan.run().outputs()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.y.zero_()
        with torch.cuda.graph(g, stream=s):
            plan.run()
    torch.cuda.current_stream().wait_stream(s)
    plan.y.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, plan.outputs()):
        assert torch.equal(a, b)


def test_errors(V):
    from adaptive_voice_conversion_b200 import _lib as L
    voc = V.Vocoder(n_mels=80)
    with pytest.raises(ValueError, match="samples"):
        voc.wav_to_mel([dev(utterance(1000, 0, silence=(0, 0)))])
    with pytest.raises(ValueError, match="after trimming"):    # a click at the end trims [512, 1100): 588 samples
        y = np.zeros(1100, np.float32)
        y[1090:] = 1.0
        voc.wav_to_mel([dev(y)])
    with pytest.raises(ValueError, match="frames"):
        voc.mel_to_wav([dev(np.full((4, 80), 0.5, np.float32))])
    with pytest.raises(ValueError, match=r"\[T, 80\]"):
        voc.mel_to_wav([dev(np.full((40, 512), 0.5, np.float32))])
    with pytest.raises(L.AvcError, match="n_fft"):
        V.stft([dev(utterance(5000, 0))], V.AudioParams(n_fft=1024))
    with pytest.raises(L.AvcError, match="hop"):
        V.stft([dev(utterance(5000, 0))], V.AudioParams(hop_length=1300))


@pytest.fixture()
def conversion_files(tmp_path):
    cfg = orc.default_config(80)
    cfg_path = tmp_path / "config.yaml"
    cfg_path.write_text(yaml.safe_dump(cfg))
    ckpt = tmp_path / "model.ckpt"
    torch.save(orc.init_state(cfg, seed=0), ckpt)
    attr = tmp_path / "attr.pkl"
    with open(attr, "wb") as f:
        pickle.dump({"mean": np.full(80, 0.4, np.float32), "std": np.full(80, 0.2, np.float32)}, f)
    src, tgt = tmp_path / "src.wav", tmp_path / "tgt.wav"
    wavfile.write(src, SR, utterance(30000, 90))
    wavfile.write(tgt, SR, utterance(24000, 91))
    return cfg, types.SimpleNamespace(config=str(cfg_path), model=str(ckpt), attr=str(attr), source=str(src),
                                      target=str(tgt), output=str(tmp_path / "out.wav"), sample_rate=SR)


def check_wav(path):
    rate, wav = wavfile.read(path)
    assert rate == SR and wav.dtype == np.float32 and wav.ndim == 1 and len(wav) > 0
    assert np.isfinite(wav).all()


def test_inference_cli_wav_to_wav(conversion_files):
    _, a = conversion_files
    r = subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), "-c", a.config, "-m", a.model, "-a", a.attr,
                        "-s", a.source, "-t", a.target, "-o", a.output], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    check_wav(a.output)


def test_inferencer_inference_from_path_with_vocoder(conversion_files, V):
    from adaptive_voice_conversion_b200.inference import Inferencer
    cfg, a = conversion_files
    inf = Inferencer(cfg, a, vocoder=V.Vocoder(n_mels=80))
    inf.inference_from_path()
    check_wav(a.output)
