"""float64 restatement of the PGHI start phase of avc_pghi (csrc/audio.cu): Phase Gradient Heap Integration
(Prusa, Balazs & Sondergaard 2017) run frame by frame with the whole magnitude known (RTPGHI, Prusa & Holighaus 2017),
on the STFT of oracle/audio_oracle.py (frame f centred on sample f * hop, the Hann window centred in the n_fft frame,
phases relative to the frame start).

``pghi_heap`` is the definition: the literal heap algorithm, written with heapq over tuples.  ``pghi_scan`` restates it
as the kernel computes it -- directional widest-path levels by scans of clamp maps, segmented arg-max seeds, segmented
prefix sums of the phase steps -- vectorised over frames in numpy (Hillis-Steele scans).  Shared by
tests/test_vocoder_pghi_host.py (formulas, worked examples, scan against heap) and tests/test_gpu_vocoder_pghi.py
(the kernel against the heap)."""
import heapq

import numpy as np

import oracle.audio_oracle as ao

GAMMA = 0.25645          # Gaussian approximation of the Hann window: lambda = GAMMA * win^2 samples^2
TOL = 1e-5               # default significance threshold, relative to the utterance's largest magnitude; not tuned
NONE, TIME, LEFT, RIGHT, SEED = 0, 1, 2, 3, 4   # parent codes (AVC_PGHI_*)
_ISLAND = 5


def derivatives(S, tol=TOL, n_fft=ao.N_FFT, hop=ao.HOP, win=ao.WIN):
    """(dt, dk, sig) for magnitudes S [F, K]: the phase advance per frame dt(f,k) = hop ((N/lambda) d_k l + 2 pi k/N),
    the phase step per bin dk(f,k) = -(lambda/(N hop)) d_f l - pi, with l = ln max(S, tol s_max) and centred
    differences (one-sided at the edges), and the significance mask S > 0 and S >= tol s_max.  tol is rounded to
    float32, as the C entry point receives it."""
    S = np.asarray(S, np.float64)
    thr = float(np.float32(tol)) * float(S.max())
    sig = (S > 0) & (S >= thr)
    lam = GAMMA * win * win
    F, K = S.shape
    k = np.arange(K)[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):   # l = -inf only where s_max = 0: nothing is significant
        ell = np.log(np.maximum(S, thr))
        d_k = np.gradient(ell, axis=1) if K > 1 else np.zeros_like(ell)
        d_f = np.gradient(ell, axis=0) if F > 1 else np.zeros_like(ell)
        dt = hop * ((n_fft / lam) * d_k + 2 * np.pi * k / n_fft)
        dk = -(lam / (n_fft * hop)) * d_f - np.pi
    return dt, dk, sig


def wrap(phi):
    """phi wrapped to (-pi, pi]."""
    return np.pi - np.mod(np.pi - phi, 2 * np.pi)


# ------------------------------------------------------------------ the definition
def heap_frame(s_prev, sig_prev, s_cur, sig_cur, phi_prev=None, dt_prev=None, dt_cur=None, dk_cur=None):
    """(parent, phi) of one frame by the literal heap algorithm.  Keys pop larger magnitude first, then frame f-1
    before frame f, then the lower bin.  The phase inputs default to zero (parents only)."""
    K = len(s_cur)
    z = np.zeros(K)
    phi_prev, dt_prev, dt_cur, dk_cur = [z if v is None else np.asarray(v, np.float64)
                                         for v in (phi_prev, dt_prev, dt_cur, dk_cur)]
    parent, phi, done = np.zeros(K, np.int8), np.zeros(K), np.zeros(K, bool)
    heap = [(-float(s_prev[k]), 0, k) for k in range(K) if sig_prev[k]]
    heapq.heapify(heap)
    while True:
        while heap:
            _, fr, k = heapq.heappop(heap)
            if fr == 0:
                if sig_cur[k] and not done[k]:
                    phi[k] = phi_prev[k] + 0.5 * (dt_prev[k] + dt_cur[k])
                    parent[k], done[k] = TIME, True
                    heapq.heappush(heap, (-float(s_cur[k]), 1, k))
                continue
            for n, sign, code in ((k - 1, -1.0, RIGHT), (k + 1, 1.0, LEFT)):
                if 0 <= n < K and sig_cur[n] and not done[n]:
                    phi[n] = phi[k] + sign * 0.5 * (dk_cur[k] + dk_cur[n])
                    parent[n], done[n] = code, True
                    heapq.heappush(heap, (-float(s_cur[n]), 1, n))
        left = np.flatnonzero(np.asarray(sig_cur, bool) & ~done)
        if left.size == 0:
            return parent, phi
        k = int(left[np.argmax(np.asarray(s_cur, np.float64)[left])])   # the first of equal maxima: the lower bin
        parent[k], done[k] = SEED, True
        heapq.heappush(heap, (-float(s_cur[k]), 1, k))


def _integrate(S, tol, frame_fn, n_fft, hop, win):
    S = np.asarray(S, np.float64)
    dt, dk, sig = derivatives(S, tol, n_fft, hop, win)
    F, K = S.shape
    phi, parent = np.zeros((F, K)), np.zeros((F, K), np.int8)
    zs, zb = np.zeros(K), np.zeros(K, bool)
    for f in range(F):
        p = f - 1
        parent[f], phi[f] = frame_fn(S[p] if f else zs, sig[p] if f else zb, S[f], sig[f],
                                     phi[p] if f else zs, dt[p] if f else zs, dt[f], dk[f])
    return wrap(phi), parent


def pghi_heap(S, tol=TOL, n_fft=ao.N_FFT, hop=ao.HOP, win=ao.WIN):
    """(phi wrapped to (-pi, pi], parent) [F, K] of magnitudes S [F, K]: the heap integration, frame by frame."""
    return _integrate(S, tol, heap_frame, n_fft, hop, win)


def pghi(S, tol=TOL, n_fft=ao.N_FFT, hop=ao.HOP, win=ao.WIN):
    """The start spectrum S e^{i phi} (complex128)."""
    phi, _ = pghi_heap(S, tol, n_fft, hop, win)
    return np.asarray(S, np.float64) * np.exp(1j * phi)


# ------------------------------------------------------------------ the scan restatement
def keys(s_prev, sig_prev, s_cur, sig_cur):
    """(a, c) int64 [B, K]: the rank of each significant entry of frames f-1 and f in the heap's pop order (larger
    pops first), 0 for an insignificant one."""
    s_prev, s_cur = np.atleast_2d(s_prev).astype(np.float64), np.atleast_2d(s_cur).astype(np.float64)
    B, K = s_cur.shape
    s = np.concatenate([s_prev, s_cur], axis=1)
    fr = np.concatenate([np.zeros((B, K)), np.ones((B, K))], axis=1)
    k = np.tile(np.arange(K), 2)[None, :].repeat(B, 0)
    order = np.lexsort((-k, -fr, s), axis=-1)        # ascending: the last entry pops first
    rank = np.empty((B, 2 * K), np.int64)
    np.put_along_axis(rank, order, np.arange(1, 2 * K + 1)[None, :].repeat(B, 0), axis=1)
    sig = np.concatenate([np.atleast_2d(sig_prev), np.atleast_2d(sig_cur)], axis=1).astype(bool)
    rank = np.where(sig, rank, 0)
    return rank[:, :K], rank[:, K:]


def _scan(op, ident, x, reverse=False):
    """Inclusive Hillis-Steele scan along the last axis of the tuple of arrays x with the associative op(earlier,
    later); reverse scans from the last element down."""
    if reverse:
        return tuple(v[..., ::-1] for v in _scan(op, ident, tuple(v[..., ::-1] for v in x)))
    K, d = x[0].shape[-1], 1
    while d < K:
        prev = tuple(np.concatenate([np.full(v.shape[:-1] + (d,), i, v.dtype), v[..., :-d]], axis=-1)
                     for v, i in zip(x, ident))
        x = op(prev, x)
        d *= 2
    return x


_BIG = np.iinfo(np.int64).max


def _clamp(e, l):      # x -> min(max(x, lo), hi): apply e, then l
    return (np.minimum(np.maximum(e[0], l[0]), l[1]), np.minimum(np.maximum(e[1], l[0]), l[1]))


def _segmax(e, l):     # (starts a segment, key)
    return (e[0] | l[0], np.where(l[0], l[1], np.maximum(e[1], l[1])))


def _segsum(e, l):     # (starts a segment, value)
    return (e[0] | l[0], np.where(l[0], l[1], e[1] + l[1]))


def _shift(v, d, fill):
    """v moved d places along the last axis (d > 0: toward higher index), filled with fill."""
    out = np.full_like(v, fill)
    if d > 0:
        out[..., d:] = v[..., :-d]
    else:
        out[..., :d] = v[..., -d:]
    return out


def scan_parents(a, c):
    """Parents [B, K] from the keys (a of frame f-1, c of frame f; 0 = insignificant) as the kernel computes them:
    L_k = max(a_k, min(L_{k-1}, c_{k-1})) and R_k = max(a_k, min(R_{k+1}, c_{k+1})) as scans of clamp maps; the
    parent is the largest of the time candidate a_k (checked first), min(L_{k-1}, c_{k-1}) and min(R_{k+1}, c_{k+1});
    a significant bin with none is seeded by a segmented arg-max over its run."""
    a, c = np.asarray(a, np.int64), np.asarray(c, np.int64)
    c_l, c_r = _shift(c, 1, 0), _shift(c, -1, 0)
    L, _ = _scan(_clamp, (0, _BIG), (a, np.maximum(a, c_l)))
    R, _ = _scan(_clamp, (0, _BIG), (a, np.maximum(a, c_r)), reverse=True)
    lc = np.minimum(_shift(L, 1, 0), c_l)
    rc = np.minimum(_shift(R, -1, 0), c_r)
    par = np.where(c == 0, NONE,
                   np.where((a > 0) & (a >= lc) & (a >= rc), TIME,
                            np.where(lc > rc, LEFT, np.where(rc > lc, RIGHT, _ISLAND))))
    isl = par == _ISLAND
    reset = ~isl
    _, fw = _scan(_segmax, (False, 0), (reset, np.where(isl, c, 0)))
    _, bw = _scan(_segmax, (False, 0), (reset, np.where(isl, c, 0)), reverse=True)
    top = np.maximum(fw, bw)
    par = np.where(isl, np.where(c == top, SEED, np.where(bw == top, RIGHT, LEFT)), par)
    return par.astype(np.int8)


def scan_frame(s_prev, sig_prev, s_cur, sig_cur, phi_prev, dt_prev, dt_cur, dk_cur):
    """(parent, phi) of one frame (or a batch of frames [B, K]) by the scans: roots are time steps and seeds, the
    left-parented chains are a forward segmented sum of (dk_{k-1} + dk_k)/2, the right-parented ones a backward
    segmented sum of -(dk_{k+1} + dk_k)/2."""
    a, c = keys(s_prev, sig_prev, s_cur, sig_cur)
    par = scan_parents(a, c)
    dt_prev, dt_cur, dk = (np.atleast_2d(v).astype(np.float64) for v in (dt_prev, dt_cur, dk_cur))
    phi_prev = np.atleast_2d(phi_prev).astype(np.float64)
    root = np.where(par == TIME, phi_prev + 0.5 * (dt_prev + dt_cur), 0.0)
    inc_l = 0.5 * (_shift(dk, 1, 0.0) + dk)
    inc_r = -0.5 * (_shift(dk, -1, 0.0) + dk)
    _, fw = _scan(_segsum, (False, 0.0), (par != LEFT, np.where(par == LEFT, inc_l, root)))
    _, bw = _scan(_segsum, (False, 0.0), (par != RIGHT, np.where(par == RIGHT, inc_r, root)), reverse=True)
    phi = np.where(par == LEFT, fw, np.where(par == RIGHT, bw, root))
    if np.ndim(s_cur) == 1:
        return par[0], phi[0]
    return par, phi


def pghi_scan(S, tol=TOL, n_fft=ao.N_FFT, hop=ao.HOP, win=ao.WIN):
    """pghi_heap through the scan restatement."""
    return _integrate(S, tol, scan_frame, n_fft, hop, win)
