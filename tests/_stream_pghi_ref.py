"""float64 restatements of the streamed PGHI start (avc_pghi_stream, include/avc_b200.h) and of an RTISI-LA step whose
entering frames start from a given spectrum (avc_rtisi_la_from).

Frame f of a stream of T frames is _pghi_ref.heap_frame with the threshold tol s_max(f), s_max(f) the largest magnitude
of frames 0 .. min(f+1, T-1): l of rows f-1, f and f+1 and the significance of frames f-1 and f all use it, with
derivatives' formulas (centred differences, one-sided at the ends).  phi(f-1) is the stream's own PGHI phase.  Shared
by tests/test_stream_pghi_host.py and tests/test_gpu_stream_pghi.py."""
import numpy as np

import _pghi_ref as P
import _rtisi_ref as R


def stream_pghi(S, tol=P.TOL, hop=300, win=1200, n_fft=R.NFFT, s_max=None):
    """(phi wrapped to (-pi, pi], parent) [T, K] of a closed stream of magnitudes S [T, K].  s_max: the largest
    magnitude of the frames before S (a stream continued from them; their phases are not needed when S[0] is the
    first frame)."""
    S = np.asarray(S, np.float64)
    T, K = S.shape
    lam = P.GAMMA * win * win
    k = np.arange(K)
    tol32 = float(np.float32(tol))
    phi, parent = np.zeros((T, K)), np.zeros((T, K), np.int8)
    prev = np.zeros(K)
    run_max = 0.0 if s_max is None else float(s_max)
    for f in range(T):
        run_max = max(run_max, float(S[:min(f + 1, T - 1) + 1].max()))
        thr = tol32 * run_max
        with np.errstate(divide="ignore", invalid="ignore"):
            ell = {i: np.log(np.maximum(S[i], thr)) for i in range(max(f - 1, 0), min(f + 1, T - 1) + 1)}
            dt = {i: hop * ((n_fft / lam) * np.gradient(ell[i]) + 2 * np.pi * k / n_fft) for i in ell if i <= f}
            d_f = (np.zeros(K) if T == 1 else ell[1] - ell[0] if f == 0 else ell[f] - ell[f - 1] if f == T - 1
                   else 0.5 * (ell[f + 1] - ell[f - 1]))
            dk = -(lam / (n_fft * hop)) * d_f - np.pi
        sig = lambda i: (S[i] > 0) & (S[i] >= thr)   # noqa: E731
        if f:
            parent[f], phi[f] = P.heap_frame(S[f - 1], sig(f - 1), S[f], sig(f), prev, dt[f - 1], dt[f], dk)
        else:
            parent[f], phi[f] = P.heap_frame(np.zeros(K), np.zeros(K, bool), S[0], sig(0), None, None, dt[0], dk)
        prev = phi[f]
    return P.wrap(phi), parent


def stream_X(S, **kw):
    """The start spectra S e^{i phi} (complex128) of stream_pghi."""
    phi, _ = stream_pghi(S, **kw)
    return np.asarray(S, np.float64) * np.exp(1j * phi)


def step_from(st, X, mags, close, n_iter, deemph=0.0):
    """_rtisi_ref.step with each entering frame's windowed inverse frame window x irfft(X row) (imaginary parts of the
    DC and Nyquist bins ignored) instead of the projection of the estimate."""
    out = []
    off = (R.NFFT - st.win) // 2
    w = R.hann(st.win)
    for x, m in zip(X, mags):
        T = st.c + st.nbuf
        st.mag[T] = np.asarray(m, np.float64)
        x = np.array(x, np.complex128)
        x[0], x[-1] = x[0].real, x[-1].real
        st.fr[T] = np.fft.irfft(x, R.NFFT)[off:off + st.win] * w
        st.nbuf += 1
        R._iterate(st, n_iter)
        if st.nbuf == st.nb:
            R._commit(st, deemph, out)
    out += list(R.step(st, [], close, n_iter, deemph)) if close else []
    return np.asarray(out)


def rtisi_from(X, mags, win, hop, lookahead, n_iter, deemph=0.0):
    """A whole closed stream through step_from: hop (T - 1) samples."""
    return step_from(R.State(win, hop, lookahead), X, mags, True, n_iter, deemph)
