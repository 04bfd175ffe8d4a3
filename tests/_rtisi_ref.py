"""Float64 restatement of RTISI-LA as avc_rtisi_la runs it (include/avc_b200.h): one stream's state and its steps.

Sample n sits at frame n / hop; frame F covers 0 <= n - F hop + win/2 < win.  State: c committed frames, the buffered
frames c .. c + nbuf - 1 (their windowed inverse frames and magnitudes), the numerator of the committed frames over
samples c hop - win/2 ... c hop + win/2 - 1, the de-emphasis carry.
"""
import numpy as np

NFFT = 2048


def hann(win):
    """The kernels' periodic Hann, 0.5 - 0.5 cospif(2q / win) with the argument and the result in float32: the cosine
    of the float32 argument rounded to float32 (cospif is within about 1 ulp of it), then 0.5 - 0.5 c in float32.  Near
    its ends 0.5 - 0.5 c cancels, and the estimate divides by the window sum-square there, so the restatement takes
    these values rather than float64 ones."""
    x = (np.float32(2) * np.arange(win, dtype=np.float32)) / np.float32(win)
    c = np.cos(np.pi * x.astype(np.float64)).astype(np.float32)
    return (np.float32(0.5) - np.float32(0.5) * c).astype(np.float64)


class State:
    def __init__(self, win, hop, lookahead):
        self.win, self.hop, self.nb = win, hop, lookahead + 1
        self.c, self.nbuf, self.carry = 0, 0, 0.0
        self.fr, self.mag = {}, {}
        self.num = np.zeros(win)

    def copy(self):
        s = State(self.win, self.hop, self.nb - 1)
        s.c, s.nbuf, s.carry = self.c, self.nbuf, self.carry
        s.fr = {k: v.copy() for k, v in self.fr.items()}
        s.mag = {k: v.copy() for k, v in self.mag.items()}
        s.num = self.num.copy()
        return s


def _covering(n, win, hop):
    h = win // 2
    return (n + h - win) // hop + 1, (n + h) // hop


def _wss(n, lo_frame, hi_frame, win, hop):
    """Window sum-square at samples n (an array) of the frames lo_frame .. hi_frame that cover each, added in
    increasing frame order (the kernel's)."""
    w2 = hann(win) ** 2
    out = np.zeros(len(n))
    if len(n) == 0:
        return out
    h = win // 2
    first, last = _covering(int(n[0]), win, hop)[0], _covering(int(n[-1]), win, hop)[1]
    for F in range(max(lo_frame, first), min(hi_frame, last) + 1):
        q = n - F * hop + h
        m = (q >= 0) & (q < win)
        out[m] += w2[q[m]]
    return out


def estimate(st, n0, length, newest):
    win, hop, h = st.win, st.hop, st.win // 2
    a0 = st.c * hop - h
    n = n0 + np.arange(length, dtype=np.int64)
    out = np.zeros(length)
    m = (n - a0 >= 0) & (n - a0 < win)
    out[m] = st.num[(n - a0)[m]]
    for F in range(st.c, st.c + st.nbuf):
        q = n - F * hop + h
        m = (q >= 0) & (q < win)
        out[m] += st.fr[F][q[m]]
    wss = _wss(n, 0, newest, win, hop)
    return np.where(wss > np.finfo(np.float32).tiny, out / np.where(wss > 0, wss, 1.0), out)


def project(e, mag, win):
    """STFT of the windowed estimate, mag with its phase (phase 0 where |E| = 0), iSTFT times the window."""
    w = hann(win)
    off = (NFFT - win) // 2
    frame = np.zeros(NFFT)
    frame[off:off + win] = w * e
    E = np.fft.rfft(frame)
    a = np.abs(E)
    u = np.where(a > 0, E / np.where(a > 0, a, 1.0), 1.0)
    return np.fft.irfft(np.asarray(mag, np.float64) * u, NFFT)[off:off + win] * w


def _iterate(st, n_iter):
    for _ in range(n_iter):
        n0 = st.c * st.hop - st.win // 2
        est = estimate(st, n0, (st.nbuf - 1) * st.hop + st.win, st.c + st.nbuf - 1)
        new = {}
        for b in range(st.nbuf):
            F = st.c + b
            new[F] = project(est[b * st.hop:b * st.hop + st.win], st.mag[F], st.win)
        st.fr.update(new)


def _release(st, n0, length, last, deemph, out):
    win, hop, h = st.win, st.hop, st.win // 2
    a0 = st.c * hop - h
    n = n0 + np.arange(length, dtype=np.int64)
    wss = _wss(n, 0, last, win, hop)
    num = st.num[n - a0]
    x = np.where(wss > np.finfo(np.float32).tiny, num / np.where(wss > 0, wss, 1.0), num)
    for v in x[n >= 0]:       # the de-emphasis recurrence, in sample order
        st.carry = v + deemph * st.carry
        out.append(st.carry)


def _commit(st, deemph, out):
    st.num = st.num + st.fr[st.c]
    _release(st, st.c * st.hop - st.win // 2, st.hop, st.c, deemph, out)
    st.num = np.concatenate([st.num[st.hop:], np.zeros(st.hop)])
    st.fr.pop(st.c)
    st.mag.pop(st.c)
    st.c += 1
    st.nbuf -= 1


def step(st, mags, close, n_iter, deemph=0.0):
    """One launch for one stream: the new frames' magnitudes mags ([p, n_bins], p may be 0), then close.  Updates st
    in place and returns the released samples."""
    out = []
    for m in mags:
        T = st.c + st.nbuf
        st.mag[T] = np.asarray(m, np.float64)
        e = estimate(st, T * st.hop - st.win // 2, st.win, T - 1)
        st.fr[T] = project(e, st.mag[T], st.win)
        st.nbuf += 1
        _iterate(st, n_iter)
        if st.nbuf == st.nb:
            _commit(st, deemph, out)
    if close:
        T = st.c + st.nbuf
        while st.nbuf > 0:
            _iterate(st, n_iter)
            _commit(st, deemph, out)
        n0, n1 = T * st.hop - st.win // 2, (T - 1) * st.hop
        if T > 0 and n1 > max(n0, 0):
            _release(st, n0, n1 - n0, T - 1, deemph, out)
    return np.asarray(out)


def rtisi(mags, win, hop, lookahead, n_iter, deemph=0.0):
    """A whole stream of magnitudes [T, n_bins], closed: hop (T - 1) samples."""
    st = State(win, hop, lookahead)
    return step(st, mags, True, n_iter, deemph)


def stft_mag(y, win, hop):
    """|STFT| (center, reflect padding, periodic Hann of win centred in n_fft) of y: [1 + len/hop, n_bins]."""
    w = np.zeros(NFFT)
    off = (NFFT - win) // 2
    w[off:off + win] = hann(win)
    yp = np.pad(np.asarray(y, np.float64), NFFT // 2, mode="reflect")
    T = 1 + len(y) // hop
    return np.abs(np.stack([np.fft.rfft(yp[f * hop:f * hop + NFFT] * w) for f in range(T)]))


def spectral_convergence(S, y, win, hop):
    """||S - |STFT(y)||| / ||S|| over the frames of y's grid."""
    A = stft_mag(y, win, hop)
    T = min(len(A), len(S))
    return float(np.linalg.norm(S[:T] - A[:T]) / np.linalg.norm(S[:T]))


def harmonic(n, sr, f0s=(140.0, 220.0), seed=0):
    """A seeded synthetic voiced signal: harmonics of a slowly gliding f0, with a little noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    y = np.zeros(n)
    for f0 in f0s:
        f = f0 * (1.0 + 0.05 * np.sin(2 * np.pi * 1.3 * t))
        ph = 2 * np.pi * np.cumsum(f) / sr
        for k in range(1, 12):
            y += np.sin(k * ph + rng.uniform(0, 2 * np.pi)) / k
    return 0.1 * y / np.abs(y).max() + 1e-3 * rng.standard_normal(n)
