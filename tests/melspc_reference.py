# -*- coding: utf-8 -*-
"""Float64 numpy restatement of the reference's melspc feature extraction (bin/feature_extract.py
``melspectrogram_extract``: low-cut FIR, ``librosa.feature.melspectrogram(x / 32768, power=1.0)`` in librosa 0.6.2-0.9's
semantics, ``np.float32(np.log10(np.maximum(1e-10, mspc.T)))``), written independently of
``pytorchwavenetvocoder_b200/utils/melspc.py``: ``np.pad``, ``np.fft.rfft``, ``np.abs``, its own filterbank code,
``np.log10``, ``np.float32``.  librosa is not installed, so it is unpinned against librosa; tests/test_melspc_host.py pins
it by what the pieces are (documented mel-scale values, filter peaks and areas, a bin-centred cosine, Parseval, scipy's
``lfilter``).  ``feature_bounds`` gives the element-wise interval the GPU's float32 features must round from (derived in
its docstring)."""
import numpy as np

U = 2.0 ** -53      # unit roundoff of float64
EPS = 1e-10


# ---- the filterbank, restated (librosa.filters.mel with htk=False, norm=1, dtype=float32) ----------------------------
def slaney_hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return np.where(f >= 1000.0, 1000.0 / (200.0 / 3) + np.log(f / 1000.0) / (np.log(6.4) / 27.0), f / (200.0 / 3))


def slaney_mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    return np.where(m >= 1000.0 / (200.0 / 3), 1000.0 * np.exp((np.log(6.4) / 27.0) * (m - 1000.0 / (200.0 / 3))),
                    (200.0 / 3) * m)


def mel_basis(fs, fftl, n_mels, fmin, fmax):
    """(n_mels, fftl // 2 + 1) float32: triangles between consecutive Slaney mel points over the rfft bin frequencies,
    each stored as float32 and then scaled by 2 / (f[i + 2] - f[i]) (float64 product rounded back to float32)."""
    bins = np.linspace(0, float(fs) / 2, fftl // 2 + 1, endpoint=True)
    edges = slaney_mel_to_hz(np.linspace(slaney_hz_to_mel(float(fmin)), slaney_hz_to_mel(float(fmax)), n_mels + 2))
    width = np.diff(edges)
    dist = edges[:, None] - bins[None, :]
    rising = -dist[:-2] / width[:-1, None]
    falling = dist[2:] / width[1:, None]
    tri = np.maximum(0, np.minimum(rising, falling)).astype(np.float32)
    return (tri * (2.0 / (edges[2:] - edges[:-2]))[:, None]).astype(np.float32)


# ---- the signal path -----------------------------------------------------------------------------------------------
def lowcut(x, taps):
    """lfilter(taps, 1, x) with zero initial state, as sum_k taps[k] x[n - k] in ascending k, and the per-sample bound
    sum_k |taps[k] x[n - k]| used for the error bars."""
    x = np.asarray(x, dtype=np.float64)
    y = np.zeros_like(x)
    mag = np.zeros_like(x)
    for k, b in enumerate(taps):
        if k >= len(x):
            break
        y[k:] += b * x[:len(x) - k]
        mag[k:] += abs(b) * np.abs(x[:len(x) - k])
    return y, mag


def fir_bound(mag, n_taps=255):
    """|GPU - oracle| bound of the filtered float64 signal: sum_k |b_k x_{n-k}| * n_taps * 2^-53."""
    return mag * n_taps * U


def frames(x, fftl, hop):
    """(1 + len // hop, fftl) frames of np.pad(x, fftl // 2, mode="reflect") (librosa's center=True)."""
    xp = np.pad(np.asarray(x, dtype=np.float64), fftl // 2, mode="reflect")
    n = 1 + len(x) // hop
    idx = np.arange(n)[:, None] * hop + np.arange(fftl)[None, :]
    return xp[idx]


def hann(fftl):
    from scipy.signal import get_window
    return get_window("hann", fftl)


def magnitude(x, fftl, hop):
    """|rfft(frame * window)| of x / 32768, (frames, fftl // 2 + 1) float64."""
    return np.abs(np.fft.rfft(frames(np.asarray(x, dtype=np.float64) / 32768, fftl, hop) * hann(fftl), axis=1))


def melspc(x, fs, fftl, hop, n_mels, fmin=None, fmax=None, taps=None):
    """The features of one utterance (x in int16 units): (float32 features, float64 mel energies E, the filtered
    float64 signal, its sum_k |b_k x_{n-k}|).  ``taps`` None: no low-cut filter."""
    x = np.asarray(x, dtype=np.float64)
    if taps is not None:
        x, mag = lowcut(x, taps)
    else:
        mag = np.zeros_like(x)
    basis = mel_basis(fs, fftl, n_mels, 0 if fmin is None else fmin, fs // 2 if fmax is None else fmax)
    E = magnitude(x, fftl, hop) @ basis.astype(np.float64).T
    return np.float32(np.log10(np.maximum(EPS, E))), E, x, mag


def feature_bounds(xf, delta, E, fs, fftl, hop, n_mels, fmin=None, fmax=None):
    """Element-wise interval [lo, hi] (float64, log10 domain) that contains both the GPU's and this oracle's log10 value
    before their float32 rounding, so the GPU's float32 feature must lie in [float32(lo), float32(hi)]: equal to
    float32(oracle) unless the interval straddles a float32 rounding boundary, and then one of its two neighbours.

    xf: the oracle's filtered signal (int16 units), delta: per-sample bound of |GPU - oracle| on it (zero without the
    filter), E: the oracle's float64 mel energies.  With u = 2^-53 and L = log2(fftl), first order in u:
      * frame input a_n = x_n / 32768 * w_n: the division is exact, the product one rounding (u |a_n|); the two inputs
        differ by at most delta_n / 32768 * w_n, so D = sum_n delta_n w_n / 32768 bounds the input difference's effect
        on every bin (|twiddle| = 1);
      * FFT: a radix-2 stage rounds each butterfly output at most by eta (|a| + |b|) with eta = 4u (complex product of
        the fma form) + u/2 (correctly rounded twiddle) + sqrt(2) u (add / subtract) < 6u.  An error made at a node
        reaches X_k with gain 1, and the nodes of one stage that feed X_k have disjoint input sets, so each stage adds
        at most 6u F with F = sum_n |a_n|; pocketfft's radix-4 / radix-2 passes obey the same per-level model.  Both
        sides: |dX_k| <= 2 (1 + 6L) u F + D;
      * |X|: hypot within 2 ulp on the GPU, numpy's abs within 1 ulp: dS_k <= |dX_k| + 6u S_k;
      * mel sum: dE_m <= sum_k w_mk dS_k + (n_m + nb + 2) u sum_k w_mk S_k (the GPU's fma chain over the filter's n_m
        nonzero bins, the oracle's dense float64 dot over nb = fftl / 2 + 1 bins; the float32 table is shared exactly);
      * log10: the true value lies in [log10(max(E - dE, 1e-10)), log10(max(E + dE, 1e-10))] (this is the carried
        error divided by max(E, 1e-10) ln 10, without linearising), widened by both sides' log10 rounding: 1 ulp for
        the GPU's log10, 4 ulp for numpy's, i.e. 10 u |log10 E|."""
    fmin = 0 if fmin is None else fmin
    fmax = fs // 2 if fmax is None else fmax
    L = int(np.log2(fftl))
    w = hann(fftl)
    basis = mel_basis(fs, fftl, n_mels, fmin, fmax).astype(np.float64)
    nb = fftl // 2 + 1
    S = magnitude(xf, fftl, hop)
    F = np.abs(frames(xf / 32768, fftl, hop)) @ w
    D = frames(np.asarray(delta, dtype=np.float64) / 32768, fftl, hop) @ w
    dX = 2 * (1 + 6 * L) * U * F + D                      # (frames,)
    n_m = np.count_nonzero(basis, axis=1)                   # (n_mels,)
    wsum = basis.sum(axis=1)
    dE = (dX[:, None] + 6 * U * S.max(axis=1, keepdims=True)) * wsum[None, :] + (n_m + nb + 2)[None, :] * U * E
    lo = np.log10(np.maximum(E - dE, EPS))
    hi = np.log10(np.maximum(E + dE, EPS))
    r = 10 * U * np.abs(np.log10(np.maximum(E, EPS))) + 1e-300
    return lo - r, hi + r
