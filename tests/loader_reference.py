# -*- coding: utf-8 -*-
"""numpy restatement of ``wnb_make_train_batch`` (csrc/loader.cu), used by tests/test_gpu_loader.py and checked on the CPU
by tests/test_train_batch_adam_reference.py.

For batch row b the window starts at the absolute stream position ``so = s0 + b*hop``; every ring index is a position
modulo the ring's capacity:

    x[b][i] = enc(wave[(so + i) % cap_s])        t[b][i] = enc(wave[(so + i + 1) % cap_s])        i < T
    row     = (so // U + j) % cap_f                                  (up-sampling layer)
            = fos[(so + j) % cap_s] % cap_f                          (extend_time: frame_of_sample)
    h[b][d][j] = scaler(feat[row][d])                                j < Tf

Every operation is a single IEEE operation in a stated dtype, so the kernel must match this bit for bit.
"""
import numpy as np

# scaler arithmetic of the kernel's feat_f64 argument (and mean / scale present or NULL)
SCALER_MODES = ("f64", "f64_none", "mode0", "mode2", "f32_none")


def scaler_mode_args(mode):
    """(feature dtype, feat_f64 argument, whether mean / scale are passed) of a scaler mode"""
    return {"f64": (np.float64, 1, True), "f64_none": (np.float64, 1, False), "mode0": (np.float32, 0, True),
            "mode2": (np.float32, 2, True), "f32_none": (np.float32, 0, False)}[mode]


def apply_scaler(v, mean, scale, mode):
    """StandardScaler.transform of rows v (..., D) in the arithmetic of `mode`, as float32:
    f64: float64 features, float32((v - mean) / scale);
    mode0 (scikit-learn 0.22): float32(float64(float32(float64(v) - mean)) / scale);
    mode2 (scikit-learn >= 1.x): float32 arithmetic with mean and scale cast to float32 first;
    *_none: no scaler, the value itself as float32."""
    if mode == "f64":
        assert v.dtype == np.float64
        return ((v - mean) / scale).astype(np.float32)
    if mode == "mode0":
        assert v.dtype == np.float32
        c = (v.astype(np.float64) - mean).astype(np.float32)
        return (c.astype(np.float64) / scale).astype(np.float32)
    if mode == "mode2":
        assert v.dtype == np.float32
        return (v - mean.astype(np.float32)) / scale.astype(np.float32)
    assert mode in ("f64_none", "f32_none")
    return v.astype(np.float32)


def mulaw_f32_reference(x32, mu):
    """encode_mu_law (reference wavenet.py:17-30) of float32 samples with a correctly rounded float32 log: the float32
    part (1 + mu|x|, log, sign) in float32, the division by log(1 + mu) and the rest in float64 (NEP 50 promotion).
    The log is taken in float64 and rounded once, as csrc/loader.cu and csrc/elementwise.cu do."""
    m = np.float32(mu - 1)
    x32 = np.asarray(x32, dtype=np.float32)
    arg = np.float32(1) + m * np.abs(x32)
    lg = np.log(arg.astype(np.float64)).astype(np.float32)
    num = np.sign(x32) * lg
    fx = num.astype(np.float64) / np.log(1.0 + (mu - 1))
    return np.floor((fx + 1.0) / 2.0 * float(mu - 1) + 0.5).astype(np.int64)


def mulaw_edges(mu):
    """quantiser edges of encode_mu_law with mu levels (the x where (fx + 1) / 2 * (mu - 1) + 0.5 is an integer)"""
    m = mu - 1
    fx = (np.arange(1, mu) - 0.5) / m * 2 - 1
    return np.sign(fx) / m * ((1.0 + m) ** np.abs(fx) - 1)


def mulaw_near_edges(mu):
    """float32 values on and one ulp either side of every quantiser edge"""
    e32 = mulaw_edges(mu).astype(np.float32)
    return np.concatenate([np.nextafter(e32, np.float32(-2)), e32, np.nextafter(e32, np.float32(2))])


def mulaw_edge_mask_mu(x32, mu):
    """tests/golden/cases.py mulaw_edge_mask for any mu: within 2 ulp of a quantiser edge, where numpy's SIMD float32
    log (not correctly rounded) may pick the neighbouring code"""
    e = mulaw_edges(mu)
    x = np.asarray(x32, dtype=np.float32)
    x64 = x.astype(np.float64)
    k = np.clip(np.searchsorted(e, x64), 1, len(e) - 1)
    d = np.minimum(np.abs(x64 - e[k - 1]), np.abs(x64 - e[k]))
    return d <= 2 * np.spacing(np.abs(x)).astype(np.float64)


def rows_of(so, U, Tf, cap_s, cap_f, fos):
    """feature-ring rows read by the window starting at absolute sample `so`"""
    j = np.arange(Tf, dtype=np.int64)
    if fos is None:
        return (so // U + j) % cap_f
    return fos[(so + j) % cap_s].astype(np.int64) % cap_f


def make_train_batch(codes, feat, fos, s0, hop, U, cap_s, cap_f, mean, scale, B, T, Tf, mode):
    """(x, t, h) of one wnb_make_train_batch launch.  `codes` is the mu-law code of every wave-ring slot (the encoder is
    applied per slot, so it is a gather here); `feat` is the (cap_f, D) feature ring in the dtype of `mode`."""
    D = feat.shape[1]
    x = np.empty((B, T), np.int64)
    t = np.empty((B, T), np.int64)
    h = np.empty((B, D, Tf), np.float32)
    i = np.arange(T + 1, dtype=np.int64)
    for b in range(B):
        so = s0 + b * hop
        q = codes[(so + i) % cap_s]
        x[b], t[b] = q[:-1], q[1:]
        h[b] = apply_scaler(feat[rows_of(so, U, Tf, cap_s, cap_f, fos)], mean, scale, mode).T
    return x, t, h


def ring_case(name):
    """Ring geometry of the named kernel case: dict(fos, U, T, Tf, D, B, hop, cap_s, cap_f, s0, reaches); `reaches` lists
    the edges it is built to reach (asserted through windows_reach).  fos: extend_time mode (rows through
    frame_of_sample, Tf = T); otherwise the up-sampling layer's Tf = T / U."""
    c = dict(RING_CASES[name])
    c.setdefault("D", 28)
    c.setdefault("U", 80)
    c["Tf"] = c["T"] if c["fos"] else c["T"] // c["U"]
    return c


RING_CASES = {
    # up-sampling, s0 and hop multiples of U as in the generator; the first window ends exactly at cap_s - 1, the rest
    # straddle the end by 80, 160, ... samples; 13 feature rows wrap at another window than the 1 041 samples
    "up_end_at_cap_minus_1": dict(fos=False, T=800, B=6, hop=80, cap_s=1041, cap_f=13, s0=240 + 2 * 1041 * 80,
                                  reaches=["end_at_cap_minus_1", "straddle_s", "straddle_f", "wrapped_s"]),
    # the first window's last target is slot 0 (it ends at cap_s)
    "up_end_at_cap": dict(fos=False, T=800, B=5, hop=160, cap_s=1040, cap_f=11, s0=240 + 80 * 1040,
                          reaches=["end_at_cap", "straddle_s", "straddle_f", "wrapped_s"]),
    # cap_s = T + 1, the smallest capacity the kernel accepts: every row reads every slot once; cap_f = Tf
    "up_cap_T_plus_1": dict(fos=False, T=640, B=7, hop=240, cap_s=641, cap_f=8, s0=641 * 80 * 3 + 160,
                            reaches=["straddle_s", "straddle_f", "every_slot"]),
    # extend_time: rows through frame_of_sample; windows at every offset around the end, incl. ending at cap_s - 1 and
    # at cap_s, and unwrapped ones
    "fos_offsets": dict(fos=True, T=300, B=9, hop=1, cap_s=307, cap_f=300, s0=5 * 307 + 3,
                        reaches=["end_at_cap_minus_1", "end_at_cap", "straddle_s", "inside_s", "straddle_f"]),
    "fos_cap_T_plus_1": dict(fos=True, T=256, B=4, hop=97, cap_s=257, cap_f=256, s0=257 * 11 + 3,
                             reaches=["straddle_s", "every_slot", "straddle_f"]),
    # hop = 0: every row reads the same (straddling) window
    "up_hop0": dict(fos=False, T=400, B=3, hop=0, cap_s=450, cap_f=6, s0=80 * 4 * 450 + 160,
                    reaches=["straddle_s", "straddle_f", "same_rows"]),
    # s0 >= 2^32 (int64 position arithmetic), a multiple of U
    "up_s0_above_2p32": dict(fos=False, T=800, B=4, hop=320, cap_s=1237, cap_f=17, s0=80 * 53687092,
                             reaches=["s0_2p32", "straddle_s", "straddle_f"]),
    "fos_s0_above_2p32": dict(fos=True, T=500, B=3, hop=111, cap_s=613, cap_f=509, s0=(1 << 32) + 77,
                              reaches=["s0_2p32", "straddle_s", "straddle_f"]),
}


def fos_ring(c, f0=123456789):
    """frame_of_sample ring as the generator leaves it: slot k holds the absolute frame (f0 + p // U) of the latest
    position p == k (mod cap_s) written before the last window's end"""
    tail = c["s0"] + (c["B"] - 1) * c["hop"] + c["T"] + 1 + 5
    k = np.arange(c["cap_s"], dtype=np.int64)
    p = tail - 1 - ((tail - 1 - k) % c["cap_s"])
    return (f0 + p // c["U"]).astype(np.int32)


def windows_reach(c, fos=None):
    """the set of ring edges the windows of case c reach (fos: its frame_of_sample ring in extend_time cases)"""
    got = set()
    T, Tf, cap_s, cap_f = c["T"], c["Tf"], c["cap_s"], c["cap_f"]
    for b in range(c["B"]):
        so = c["s0"] + b * c["hop"]
        last = so % cap_s + T                      # ring slot of the window's last target, before the wrap
        got.add({cap_s - 1: "end_at_cap_minus_1", cap_s: "end_at_cap"}.get(last, "other"))
        got.add("straddle_s" if last >= cap_s else "inside_s")
        if so >= cap_s:
            got.add("wrapped_s")
        if T + 1 == cap_s:
            got.add("every_slot")
        if so >= 1 << 32:
            got.add("s0_2p32")
        if np.any(np.diff(rows_of(so, c["U"], Tf, cap_s, cap_f, fos if c["fos"] else None)) < 0):
            got.add("straddle_f")
    if c["B"] > 1 and c["hop"] == 0:
        got.add("same_rows")
    return got
