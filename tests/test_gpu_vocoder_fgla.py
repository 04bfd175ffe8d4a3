"""GPU: fast Griffin-Lim (``momentum``) in avc_griffin_lim against its float64 restatement (tests/_fgla_ref.py), its
bit-exactness with momentum 0, its ragged-batch and graph-replay determinism, its argument errors, and wav-to-wav
conversion with -gl_momentum.

Inputs are the seeded synthetic signals of test_gpu_vocoder.py at 24 kHz."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle.audio_oracle as ao
import _fgla_ref as ref
from conftest import ROOT
from test_gpu_vocoder import SR, check_wav, conversion_files, dev, utterance  # noqa: F401 (conversion_files: fixture)

pytestmark = pytest.mark.gpu

M = 0.99


@pytest.fixture(scope="module")
def V():
    from adaptive_voice_conversion_b200 import vocoder
    return vocoder


def consistent(n, seed):
    """|STFT| of a signal: a spectrogram some signal has."""
    return np.abs(ao.stft(utterance(n, seed, silence=(0, 0))))


def test_zero_momentum_is_bitwise_the_plain_loop(V):
    from adaptive_voice_conversion_b200 import _lib as L
    S = [dev(consistent(n, 100 + i).astype(np.float32)) for i, n in enumerate([7000, 12345])]
    base = V.griffin_lim(S, n_iter=8)
    plan = V.GriffinLim(S, n_iter=8, momentum=0.0)
    assert plan.X_prev is None
    n0 = L.launch_count()
    zero = plan.run().outputs()
    assert L.launch_count() - n0 == 3 * 8 + 2
    for a, b in zip(base, zero):
        assert torch.equal(a, b)
    voc = V.Vocoder(n_mels=80)
    mels = [dev(np.random.default_rng(i).uniform(0.2, 0.8, (40 + 7 * i, 80)).astype(np.float32)) for i in range(3)]
    for a, b in zip(voc.mel_to_wav(mels, n_iter=8), voc.mel_to_wav(mels, n_iter=8, momentum=0.0)):
        assert torch.equal(a, b)


EPS32 = 5e-7   # fp32 rounding of one iteration's E, relative to its frame's peak (see the bound below)


def sensitivity(S, n_iter, m, eps=1e-7, seeds=3):
    """max |y' - y| / max |y| / eps of the float64 Griffin-Lim when every iteration's E is perturbed by seeded complex
    Gaussian noise of eps times its frame's peak: how far the iteration map carries an error of that relative size
    made in each iteration.  Linear in eps at these sizes."""
    def noise(rng):
        def perturb(E):
            pk = np.abs(E).max(axis=1, keepdims=True)
            return E + eps * pk * (rng.standard_normal(E.shape) + 1j * rng.standard_normal(E.shape))
        return perturb
    y = ref.griffin_lim(S, n_iter, m)
    dev_max = max(np.abs(ref.griffin_lim(S, n_iter, m, noise(np.random.default_rng(s))) - y).max() for s in range(seeds))
    return dev_max / np.abs(y).max() / eps


@pytest.mark.parametrize("n_iter", [1, 8])
def test_momentum_matches_the_oracle(V, n_iter):
    """Bound: the device computes each iteration's E in fp32, with an error of up to EPS32 of its frame's peak, and
    the later iterations carry that error forward.  So the waveform error after n iterations is at most EPS32 times the
    oracle's sensitivity over n iterations on this input.  EPS32 = 5e-7 is the level at which the 1e-5 bound of
    test_one_griffin_lim_iteration_matches_oracle admits one iteration on that test's magnitudes (their sensitivity
    is 17-21), and lies within the STFT's observed 1.3e-7 to 8.8e-7 of the frame peak.  A consistent spectrogram,
    started from zero phase, is more sensitive: at its first iteration some bins have |E| far below S, and their
    phase is set by small differences.  On these inputs the first iteration of plain Griffin-Lim already exceeds
    1e-5 of the peak (1.1e-5 on the H100).  Momentum makes the map 2.4-3x more sensitive by 8 iterations on these inputs."""
    from adaptive_voice_conversion_b200 import _lib as L
    S = [consistent(n, 20 + i) for i, n in enumerate([6000, 9137])]
    plan = V.GriffinLim([dev(s.astype(np.float32)) for s in S], n_iter=n_iter, momentum=M)
    plan.X_prev.fill_(float("nan"))     # the first iteration must not read it
    n0 = L.launch_count()
    got = plan.run().outputs()
    assert L.launch_count() - n0 == 3 * n_iter + 2
    for s, z in zip(S, got):
        y = ref.griffin_lim(s, n_iter, momentum=M)
        err = float(np.abs(z.cpu().numpy() - y).max() / np.abs(y).max())
        k = sensitivity(s, n_iter, M)
        print(f"momentum {M}, {n_iter} iterations, T={s.shape[0]}: max error / peak {err:.2e}; sensitivity {k:.0f}, "
              f"bound {EPS32 * k:.2e}")
        assert err < EPS32 * k, (err, k)


def test_momentum_100_iterations_tracks_the_oracle(V):
    y = utterance(SR, 30)
    S = np.abs(ao.stft(y))
    z = V.griffin_lim([dev(S.astype(np.float32))], momentum=M)[0].cpu().numpy().astype(np.float64)
    sc, sc_ref = ao.spectral_convergence(S, z), ao.spectral_convergence(S, ref.griffin_lim(S, 100, momentum=M))
    sc_plain = ao.spectral_convergence(S, ao.griffin_lim(S, 100))
    print(f"momentum {M}, 100 iterations: spectral convergence {sc:.5f} (oracle {sc_ref:.5f}; without momentum "
          f"{sc_plain:.5f})")
    assert abs(sc - sc_ref) < 1e-3, (sc, sc_ref)


def test_momentum_batches_are_bitwise_per_utterance(V):
    S = [dev(consistent(n, 70 + i).astype(np.float32)) for i, n in enumerate([9000, 15001, 9000, 20000])]
    batch = V.griffin_lim(S, n_iter=10, momentum=M)
    again = V.griffin_lim(S, n_iter=10, momentum=M)
    for s, a, b in zip(S, batch, again):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)
        assert torch.equal(a, V.griffin_lim([s], n_iter=10, momentum=M)[0])
    voc = V.Vocoder(n_mels=80)
    mels = [dev(np.random.default_rng(i).uniform(0.2, 0.8, (30 + 11 * i, 80)).astype(np.float32)) for i in range(3)]
    out = voc.mel_to_wav(mels, n_iter=10, momentum=M)
    for m, a in zip(mels, out):
        assert torch.equal(a, voc.mel_to_wav([m], n_iter=10, momentum=M)[0])


def test_momentum_graph_replay_is_bitwise(V):
    S = [dev(consistent(n, 80 + i).astype(np.float32)) for i, n in enumerate([7000, 12345])]
    plan = V.GriffinLim(S, n_iter=8, momentum=M)
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
    plan.X_prev.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, plan.outputs()):
        assert torch.equal(a, b)


def test_momentum_errors_on_the_device_path(V):
    from adaptive_voice_conversion_b200 import _lib as L
    S = [dev(consistent(6000, 90).astype(np.float32))]
    n0 = L.launch_count()
    for m in (-0.1, 1.0, 2.0, float("nan"), float("inf")):
        with pytest.raises(L.AvcError, match="momentum"):
            V.griffin_lim(S, n_iter=4, momentum=m)
    plan = V.GriffinLim(S, n_iter=4, momentum=0.5)
    plan.desc.X_prev = None
    with pytest.raises(L.AvcError, match="needs X_prev"):
        plan.run()
    plan.desc.X_prev = plan.desc.X
    with pytest.raises(L.AvcError, match="overlaps X"):
        plan.run()
    plan.desc.X_prev = plan.desc.X + 8
    with pytest.raises(L.AvcError, match="overlaps X"):
        plan.run()
    assert L.launch_count() == n0
    with pytest.raises(L.AvcError, match="momentum"):
        V.Vocoder(n_mels=80).mel_to_wav([dev(np.full((40, 80), 0.5, np.float32))], momentum=1.0)
    plan = V.GriffinLim(S, n_iter=4, momentum=0.5)      # the stream is still usable
    assert torch.isfinite(plan.run().outputs()[0]).all()


def test_inference_cli_wav_to_wav_with_momentum(conversion_files):
    _, a = conversion_files
    r = subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), "-c", a.config, "-m", a.model, "-a", a.attr,
                        "-s", a.source, "-t", a.target, "-o", a.output, "-gl_momentum", "0.99", "-gl_iters", "32"],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    check_wav(a.output)
