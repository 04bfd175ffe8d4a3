"""float64 restatement of fast Griffin-Lim (Perraudin, Balazs & Sondergaard 2013) in the form of librosa's and
torchaudio's ``momentum``, on the STFT / iSTFT of oracle/audio_oracle.py.  Shared by tests/test_vocoder_fgla_host.py
(against the plain oracle loop and a worked example) and tests/test_gpu_vocoder_fgla.py (against the kernels)."""
import numpy as np

import oracle.audio_oracle as ao


def griffin_lim(S, n_iter=100, momentum=0.0, perturb=None):
    """From zero phase, with c = m / (1 + m): E = stft(istft(X)), A = E - c P (A = E the first time and whenever
    c = 0), P = E, X = S A / max(1e-8, |A|); returns istft(X).  With momentum 0 this is ao.griffin_lim bit for bit.
    perturb(E) -> E, when given, is applied to every iteration's E (the sensitivity analysis of the GPU tests)."""
    S = np.asarray(S, np.float64)
    X = S.astype(np.complex128)
    c, P = momentum / (1.0 + momentum), None
    for _ in range(n_iter):
        E = ao.stft(ao.istft(X))
        if perturb is not None:
            E = perturb(E)
        A = E if P is None or c == 0 else E - c * P
        P = E
        X = S * A / np.maximum(1e-8, np.abs(A))
    return ao.istft(X)
