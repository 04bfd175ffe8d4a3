"""GPU: the PGHI start phase (avc_pghi, ``init="pghi"``) against the float64 heap integration of tests/_pghi_ref.py
-- parents exactly, phases within a measured bound -- its ragged-batch and run-to-run determinism, its composition with
Griffin-Lim and momentum, graph replay, its effect on spectral convergence, and wav-to-wav conversion with -gl_init.

Inputs are the seeded synthetic signals of test_gpu_vocoder.py and tools/bench_vocoder.py at 24 kHz."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

import oracle.audio_oracle as ao
import _fgla_ref as fgla
import _pghi_ref as ref
from conftest import ROOT
from test_gpu_vocoder import check_wav, conversion_files, dev, utterance  # noqa: F401 (conversion_files: fixture)

pytestmark = pytest.mark.gpu

M = 0.99
# The phases are integrated in float64 from the same float32 magnitudes as the reference, so what is left is mostly
# X's float32 rounding: at most 3.5e-7 rad over the batch below on an H100 80GB HBM3 (700 W limit).
PHASE_BOUND = 2e-6


@pytest.fixture(scope="module")
def V():
    from adaptive_voice_conversion_b200 import vocoder
    return vocoder


def consistent(n_frames, seed):
    """|STFT| of a synthetic signal: a spectrogram some signal has."""
    return np.abs(ao.stft(utterance(max(ao.N_FFT // 2 + 1, ao.HOP * (n_frames - 1)), seed, silence=(0, 0))))[:n_frames]


def mel_inverse(V, n_frames, n_mels, seed):
    """The mel pseudo-inverse magnitudes mel_to_wav feeds Griffin-Lim, of a signal's mels."""
    voc = V.Vocoder(n_mels=n_mels)
    mel = ao.mel_filterbank(n_mels=n_mels) @ consistent(n_frames, seed).T
    db = 20 * np.log10(np.maximum(1e-5, mel.T))
    norm = np.clip((db - 20 + 100) / 100, 1e-8, 1).astype(np.float32)
    return voc.mel_to_mag([dev(norm)])[0].cpu().numpy()


def tied(n_frames, seed):
    """Magnitudes on three levels, with zeros: heavy ties between bins and frames, and insignificant gaps."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 4, (n_frames, 1025)).astype(np.float32) * np.float32(0.25)


LENGTHS = [1, 5, 40, 300]


@pytest.fixture(scope="module")
def batch(V):
    """[(kind, float32 magnitudes)]: every kind at every length, one ragged batch."""
    out = []
    for i, n in enumerate(LENGTHS):
        out += [("consistent", consistent(n, 10 + i).astype(np.float32)),
                ("mel80", mel_inverse(V, n, 80, 20 + i)),
                ("mel512", mel_inverse(V, n, 512, 30 + i)),
                ("tied", tied(n, 40 + i)),
                ("silent", np.zeros((n, 1025), np.float32))]
    return out


@pytest.fixture(scope="module")
def device_run(V, batch):
    mags = [dev(s) for _, s in batch]
    X, par = V.pghi(mags, parent=True)
    X2, par2 = V.pghi(mags, parent=True)
    torch.cuda.synchronize()
    return mags, X, par, X2, par2


def test_parents_and_phases_match_the_heap(batch, device_run):
    _, X, par, _, _ = device_run
    worst = 0.0
    for (kind, s), x, p in zip(batch, X, par):
        phi, want = ref.pghi_heap(s)
        got = p.cpu().numpy()
        assert np.array_equal(got, want), (kind, s.shape, np.argwhere(got != want)[:5])
        x = x.cpu().numpy()
        assert np.array_equal(np.abs(x) > 0, s > 0)
        sig = want != ref.NONE
        if kind == "silent":
            assert not sig.any() and not x.any()
            continue
        assert sig.any()
        err = float(np.abs(ref.wrap(np.angle(x[sig]) - phi[sig])).max())
        assert np.allclose(np.abs(x), s, rtol=1e-6, atol=0)
        assert np.array_equal(x[~sig].imag, np.zeros((~sig).sum(), np.float32))
        worst = max(worst, err)
        print(f"{kind} T={s.shape[0]}: max wrapped phase error {err:.2e} rad; parents "
              f"{np.bincount(want.ravel(), minlength=5).tolist()}")
    assert worst < PHASE_BOUND, worst


@pytest.mark.parametrize("win,hop", [(2048, 512), (600, 150)])
def test_parents_and_phases_match_the_heap_at_other_windows(V, win, hop):
    """λ = 0.25645 win² and the hop enter every phase step: the same kinds of magnitude as the batch above, with the
    consistent ones taken at this window and hop."""
    hp = V.AudioParams(win_length=win, hop_length=hop)
    mags = []
    for i, n in enumerate([1, 5, 40, 120]):
        y = utterance(max(1025, hop * (n - 1)), 110 + i, silence=(0, 0))
        mags += [("consistent", np.abs(ao.stft(y, ao.N_FFT, hop, win))[:n].astype(np.float32)),
                 ("mel80", mel_inverse(V, n, 80, 120 + i)), ("tied", tied(n, 130 + i)),
                 ("silent", np.zeros((n, 1025), np.float32))]
    X, par = V.pghi([dev(s) for _, s in mags], hp, parent=True)
    worst = 0.0
    for (kind, s), x, p in zip(mags, X, par):
        phi, want = ref.pghi_heap(s, hop=hop, win=win)
        got = p.cpu().numpy()
        assert np.array_equal(got, want), (kind, s.shape, np.argwhere(got != want)[:5])
        x = x.cpu().numpy()
        sig = want != ref.NONE
        if sig.any():
            worst = max(worst, float(np.abs(ref.wrap(np.angle(x[sig]) - phi[sig])).max()))
    print(f"win={win} hop={hop}: max wrapped phase error {worst:.2e} rad")
    assert worst < PHASE_BOUND, worst


def test_batches_are_bitwise_per_utterance_and_run_to_run(V, device_run):
    mags, X, par, X2, par2 = device_run
    for m, x, p, x2, p2 in zip(mags, X, par, X2, par2):
        assert torch.equal(torch.view_as_real(x), torch.view_as_real(x2)) and torch.equal(p, p2)
        (xa,), (pa,) = V.pghi([m], parent=True)
        assert torch.equal(torch.view_as_real(x), torch.view_as_real(xa)) and torch.equal(p, pa)


def test_parent_output_is_optional(V, device_run):
    mags, X, _, _, _ = device_run
    for a, b in zip(V.pghi(mags), X):
        assert torch.equal(torch.view_as_real(a), torch.view_as_real(b))


def test_start_without_iterations_is_the_istft_of_pghi(V):
    from adaptive_voice_conversion_b200 import _lib as L
    S = [dev(consistent(n, 50 + i).astype(np.float32)) for i, n in enumerate([24, 61])]
    plan = V.GriffinLim(S, n_iter=0, init="pghi")
    n0 = L.launch_count()
    y = plan.run().outputs()
    assert L.launch_count() - n0 == 3
    for a, b in zip(y, V.istft(V.pghi(S))):
        assert torch.equal(a, b)


def test_zero_start_keeps_the_old_bits_and_launches(V):
    from adaptive_voice_conversion_b200 import _lib as L
    S = [dev(consistent(n, 60 + i).astype(np.float32)) for i, n in enumerate([24, 41])]
    base = V.griffin_lim(S, n_iter=6)
    plan = V.GriffinLim(S, n_iter=6, init="zero")
    assert plan.init == "zero"
    n0 = L.launch_count()
    y = plan.run().outputs()
    assert L.launch_count() - n0 == 3 * 6 + 2
    for a, b in zip(base, y):
        assert torch.equal(a, b)
    n0 = L.launch_count()
    V.GriffinLim(S, n_iter=6, init="pghi").run()
    assert L.launch_count() - n0 == 3 * 6 + 3
    voc = V.Vocoder(n_mels=80)
    mels = [dev(np.random.default_rng(i).uniform(0.2, 0.8, (40 + 7 * i, 80)).astype(np.float32)) for i in range(2)]
    for a, b in zip(voc.mel_to_wav(mels, n_iter=6), voc.mel_to_wav(mels, n_iter=6, init="zero")):
        assert torch.equal(a, b)


def griffin_lim_from(X0, S, n_iter, momentum, perturb=None):
    """tests/_fgla_ref.griffin_lim started from the spectrum X0 instead of zero phase (n_iter >= 1).  Its first
    iteration projects E = stft(istft(X)) of the zero-phase start; substituting stft(istft(X0)) for that E makes it the
    first iteration from X0, and the loop is otherwise the reference's own.  perturb applies to every E, as there."""
    first = [True]

    def start(E):
        if first[0]:
            first[0] = False
            E = ao.stft(ao.istft(np.asarray(X0, np.complex128)))
        return E if perturb is None else perturb(E)
    assert n_iter >= 1
    return fgla.griffin_lim(S, n_iter, momentum, start)


EPS32 = 5e-7   # fp32 rounding of one iteration's E relative to its frame's peak (test_gpu_vocoder_fgla.py)


def sensitivity(X0, S, n_iter, m, eps=1e-7, seeds=3):
    """max |y' - y| / max |y| / eps of the float64 loop when every iteration's E is perturbed by seeded complex
    Gaussian noise of eps times its frame's peak (the analysis of test_gpu_vocoder_fgla.py, from X0)."""
    def noise(rng):
        def perturb(E):
            pk = np.abs(E).max(axis=1, keepdims=True)
            return E + eps * pk * (rng.standard_normal(E.shape) + 1j * rng.standard_normal(E.shape))
        return perturb
    y = griffin_lim_from(X0, S, n_iter, m)
    dev_max = max(np.abs(griffin_lim_from(X0, S, n_iter, m, noise(np.random.default_rng(s))) - y).max()
                  for s in range(seeds))
    return dev_max / np.abs(y).max() / eps


@pytest.mark.parametrize("n_iter", [1, 8])
def test_pghi_with_momentum_matches_the_oracle(V, n_iter):
    """From the float64 heap's start spectrum, with momentum: the bound of test_momentum_matches_the_oracle, one more
    iteration's worth for the float32 start spectrum."""
    S = [consistent(n, 70 + i) for i, n in enumerate([21, 31])]
    plan = V.GriffinLim([dev(s.astype(np.float32)) for s in S], n_iter=n_iter, momentum=M, init="pghi")
    plan.X_prev.fill_(float("nan"))
    got = plan.run().outputs()
    for s, z in zip(S, got):
        s32 = s.astype(np.float32).astype(np.float64)
        X0 = ref.pghi(s32)
        y = griffin_lim_from(X0, s32, n_iter, M)
        err = float(np.abs(z.cpu().numpy() - y).max() / np.abs(y).max())
        k = sensitivity(X0, s32, n_iter, M)
        print(f"pghi, momentum {M}, {n_iter} iterations, T={s.shape[0]}: max error / peak {err:.2e}; sensitivity "
              f"{k:.0f}, bound {EPS32 * (k + 1):.2e}")
        assert err < EPS32 * (k + 1), (err, k)


def test_pghi_graph_replay_is_bitwise(V):
    S = [dev(consistent(n, 80 + i).astype(np.float32)) for i, n in enumerate([24, 41])]
    plan = V.GriffinLim(S, n_iter=8, momentum=M, init="pghi")
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
    for t in (plan.y, plan.X, plan.X_prev):
        t.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, plan.outputs()):
        assert torch.equal(a, b)


def test_pghi_lowers_spectral_convergence_on_consistent_magnitudes(V):
    """On tools/bench_vocoder.py's synthetic signals (vibrato tones with harmonics and a noise floor)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_vocoder import spectral_convergence, utterances
    wavs = utterances(8, 300 * 127, seed=5)
    mags = [A for A, _ in V.magnitude(wavs)]
    for n_iter in (0, 16):
        sc = {init: float(np.median(spectral_convergence(V, mags, V.griffin_lim(mags, n_iter=n_iter, init=init))))
              for init in ("zero", "pghi")}
        print(f"{n_iter} iterations: median spectral convergence {sc}")
        assert sc["pghi"] < sc["zero"], (n_iter, sc)


def test_errors(V):
    from adaptive_voice_conversion_b200 import _lib as L
    S = [dev(consistent(24, 90).astype(np.float32))]
    n0 = L.launch_count()
    for tol in (0.0, 1.0, float("nan")):
        with pytest.raises(L.AvcError, match="tol"):
            V.pghi(S, tol=tol)
        with pytest.raises(L.AvcError, match="tol"):
            V.griffin_lim(S, V.AudioParams(pghi_tol=tol), n_iter=2, init="pghi")
    with pytest.raises(ValueError, match="init"):
        V.griffin_lim(S, n_iter=2, init="random")
    with pytest.raises(ValueError, match="bins"):
        V.pghi([S[0][:, :512]])
    for m in (1.0, float("nan")):       # checked before the PGHI start is enqueued
        with pytest.raises(L.AvcError, match="momentum"):
            V.griffin_lim(S, n_iter=2, momentum=m, init="pghi")
    plan = V.GriffinLim(S, n_iter=2, momentum=0.5, init="pghi")
    plan.desc.X_prev = None
    with pytest.raises(L.AvcError, match="needs X_prev"):
        plan.run()
    assert L.launch_count() == n0
    assert torch.isfinite(V.griffin_lim(S, n_iter=2, init="pghi")[0]).all()   # the stream is still usable


def test_inference_cli_with_pghi_start_equals_mel_to_wav(conversion_files, V):
    _, a = conversion_files
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", a.config, "-m", a.model, "-a", a.attr,
            "-s", a.source, "-t", a.target]
    mel_path = a.output[:-4] + ".npy"
    for out, extra in ((mel_path, []), (a.output, ["-gl_init", "pghi", "-gl_iters", "16"])):
        r = subprocess.run(base + ["-o", out, *extra], cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
    check_wav(a.output)
    _, wav = wavfile.read(a.output)
    want = V.Vocoder(n_mels=80).mel_to_wav([dev(np.load(mel_path).astype(np.float32))], n_iter=16, init="pghi")[0]
    assert np.array_equal(wav, want.cpu().numpy())
