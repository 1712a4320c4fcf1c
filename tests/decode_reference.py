# -*- coding: utf-8 -*-
"""Plain references for checking the decode kernels: teacher-forced float64 logits, the kernels' Philox uniforms, the
set of picks an inverse-CDF draw may legally return, and a float32 emulation of the kernels' lane-scan sampler.

Teacher forcing.  Fast generation is a causal network started from zero history, so the logits the decoder produces at
step i, given the samples it actually produced, equal the whole-sequence forward at position P-1+i of
``[padded seed | samples]`` (P = max(T0, receptive field)), with the aux upsampled and padded the same way.  One
vectorised forward replaces a step-by-step recurrence; ``forward64`` is that forward in float64 torch on any device
(matmuls, so cuBLAS DGEMM on a GPU), pinned against ``oracle.forward`` by tests/test_decode_reference.py.

The sampler (csrc/decode_warp.cu, decode_stream.cu, decode.cu).  With m = max(l), each of the 32 lanes of a warp owns
``chunk = ceil(Q/32)`` consecutive classes and sums e_q = expf(l_q - m) over them in order (lsum).  A Hillis-Steele
shuffle scan gives the lane's inclusive sum incl; total = incl of lane 31 and target = fl(uni * total).  The lane whose
interval [excl, incl) contains the target walks its classes and picks the first whose running sum from excl passes it.
Old rule: excl = incl - lsum, and no claim falls back to class Q-1.  That excl is not bit-equal to the previous lane's
incl, so [0, total) has gaps no lane claims, and a target inside one returned Q-1 (mu-law 255, a full-scale click)
whatever its probability.  Fixed rule: excl is the previous lane's incl (0 on lane 0).  The scan's sums are not
monotone in the lane (a lane of zero mass can end a rounding step above its predecessor), but every target in
[0, total) is still claimed: by the first lane whose incl exceeds it.  Overlapping claims take the lowest class.  The
walk still starts from incl - lsum and only stops at classes with e_q > 0, so a draw outside a gap picks what the old
rule picked.  A walk that never passes the target picks the last class with e_q > 0 at or before its lane (the
claiming lane itself may hold none), and a target no lane claims (>= total) the last class with e_q > 0 of the row.

Admissible picks.  The kernel's CDF differs from the float64 CDF of its own fp32 logits by: expf's <= 2 ulp per term
(4u relative, u = 2^-24), the 8-term lane sum (7u), the 5-level scan (5u), the 8-step walk inside a lane (8u), the
total's own error (<= 16u) moving the target, and the target's rounding (1u): 41u * total in all.  ``admissible``
accepts class q when e_q > 0 and its float64 interval [C_q, C_{q+1}) widened by CDF_SLACK = 64u * total contains
uni * total.
"""
import numpy as np
import torch

from oracle import wavenet_oracle as O

U24 = 2.0 ** -24
CDF_SLACK = 64 * U24          # admissible window, relative to the total (derivation above)


# ---------------------------------------------------------------------------------------------------------------------
# teacher-forced float64 logits
# ---------------------------------------------------------------------------------------------------------------------
def _conv(W, x, d=1):
    """causal conv as matmuls: W (O, C, ks), x (B, C, T) -> (B, O, T), zero history"""
    ks = W.shape[2]
    T = x.shape[2]
    y = torch.matmul(W[:, :, ks - 1], x)
    for k in range(ks - 1):
        s = (ks - 1 - k) * d
        if s < T:
            y[:, :, s:] += torch.matmul(W[:, :, k], x[:, :, :T - s])
    return y


def forward64(cfg, p, x, h, device="cpu", dtype=torch.float64):
    """``oracle.forward`` (no upsampling: h at sample rate) in float64 torch on ``device``: x (B, T) int, h (B, A, T)
    -> logits (B, T, Q) as a float64 numpy array.  ``dtype=torch.float32`` runs the same forward in plain float32 (the
    parameters and aux rounded to float32 first; on a GPU the caller keeps TF32 off), which calibrates what float32
    evaluation order alone costs against float64."""
    def t(k):
        return torch.as_tensor(np.asarray(p[k], np.float64), device=device).to(dtype)

    def b(k):
        return t(k)[None, :, None]

    W = t("causal.conv.weight")
    R, Q, ks = W.shape
    x = torch.as_tensor(np.asarray(x, np.int64), device=device) % Q
    h = torch.as_tensor(np.asarray(h, np.float64), device=device).to(dtype)
    B, T = x.shape
    out = b("causal.conv.bias").expand(B, R, T).clone()
    for k in range(ks):
        s = ks - 1 - k
        if s < T:
            out[:, :, s:] += W[:, :, k].t()[x[:, :T - s]].transpose(1, 2)
    skip = 0
    for l, d in enumerate(cfg.dilations):
        a = _conv(t("dil_sigmoid.%d.conv.weight" % l), out, d) + b("dil_sigmoid.%d.conv.bias" % l) + \
            _conv(t("aux_1x1_sigmoid.%d.weight" % l), h) + b("aux_1x1_sigmoid.%d.bias" % l)
        g = _conv(t("dil_tanh.%d.conv.weight" % l), out, d) + b("dil_tanh.%d.conv.bias" % l) + \
            _conv(t("aux_1x1_tanh.%d.weight" % l), h) + b("aux_1x1_tanh.%d.bias" % l)
        z = torch.sigmoid(a) * torch.tanh(g)
        skip = skip + _conv(t("skip_1x1.%d.weight" % l), z) + b("skip_1x1.%d.bias" % l)
        out = _conv(t("res_1x1.%d.weight" % l), z) + b("res_1x1.%d.bias" % l) + out
    r1 = torch.relu(_conv(t("conv_post_1.weight"), torch.relu(skip)) + b("conv_post_1.bias"))
    y = _conv(t("conv_post_2.weight"), r1) + b("conv_post_2.bias")
    return y.transpose(1, 2).cpu().to(torch.float64).numpy()


def teacher_forced_logits(cfg, p64, x, h, samples, device=None, chunk=None, dtype=torch.float64):
    """float64 logits (B, n, Q) the decoder should produce at steps 0..n-1, given the seed x (B, T0), the aux h as passed
    to the decoder and the samples (B, n) it produced.  Step i depends on samples[:, :i] only, so for an utterance that
    stopped at n_b < n whatever follows its n_b-th sample does not matter for steps < n_b.  ``device=None`` runs
    ``oracle.forward`` (numpy), else ``forward64`` on that device in ``dtype``, ``chunk`` utterances at a time.  The
    config's dilations are used as they are, so a config whose ``dilations`` and ``receptive_field`` were replaced
    gets the forward of those."""
    xp, hp = O._pad_inputs(cfg, p64, np.asarray(x, np.int64), np.asarray(h, np.float64))
    P = xp.shape[1]
    samples = np.asarray(samples, np.int64)
    n = samples.shape[1]
    seq = np.concatenate([xp, samples[:, :n - 1]], 1)
    hs = hp[:, :, :P - 1 + n]
    c0 = O.Config(*cfg.as_tuple()[:7] + (0,))
    c0.dilations, c0.receptive_field = list(cfg.dilations), cfg.receptive_field
    if device is None:
        assert dtype == torch.float64, "oracle.forward runs in float64 only"
        return O.forward(c0, p64, seq, hs)[:, P - 1:P - 1 + n]
    B = seq.shape[0]
    step = B if chunk is None else chunk
    return np.concatenate([forward64(c0, p64, seq[i:i + step], hs[i:i + step], device, dtype)[:, P - 1:P - 1 + n]
                           for i in range(0, B, step)], 0)


# ---------------------------------------------------------------------------------------------------------------------
# Philox4x32-10 (Salmon et al., SC'11; Random123), as the kernels draw it
# ---------------------------------------------------------------------------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 words (scalars or arrays, broadcast), key: 2 words -> 4 uint32 arrays."""
    c = [np.asarray(v, np.uint64) & _M32 for v in ctr]
    k0, k1 = [np.asarray(v, np.uint64) & _M32 for v in key]
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return [v.astype(np.uint32) for v in c]


def philox_uniform(seed, utt, step):
    """The kernels' uniform for utterance ``utt`` (batch index) at decode step ``step``: counter (step, utt, 0, 0), key
    (seed & 0xffffffff, seed >> 32), uni = (r0 >> 8) * 2^-24 in [0, 1 - 2^-24].  Broadcasts over utt and step."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    r = philox4x32_10((step, utt, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    return (r[0] >> np.uint32(8)).astype(np.float32) * np.float32(U24)


# ---------------------------------------------------------------------------------------------------------------------
# sampler: admissible set and float32 emulation
# ---------------------------------------------------------------------------------------------------------------------
def admissible(logits, uni, slack=CDF_SLACK):
    """Boolean mask (..., Q): classes an inverse-CDF draw with uniform ``uni`` (shape ...) may return from the fp32
    ``logits`` (..., Q): nonzero fp32 probability and a float64 CDF interval within ``slack * total`` of uni * total."""
    lg = np.asarray(logits, np.float32)
    m = lg.max(-1, keepdims=True)
    e32 = np.exp((lg - m).astype(np.float32))
    e = np.exp(lg.astype(np.float64) - m.astype(np.float64))
    c1 = np.cumsum(e, -1)
    c0 = c1 - e
    tot = c1[..., -1:]
    tgt = np.asarray(uni, np.float64)[..., None] * tot
    d = slack * tot
    return (e32 > 0) & (c0 - d <= tgt) & (tgt < c1 + d)


def _lane_sums(lg, chunk):
    """float32 emulation of the kernels' per-lane exponentials, lane sums and inclusive scan: (N, Q) ->
    ex (N, 32, chunk), lsum (N, 32), incl (N, 32)."""
    N, Q = lg.shape
    m = lg.max(1, keepdims=True)
    ex = np.zeros((N, 32 * chunk), np.float32)
    ex[:, :Q] = np.exp((lg - m).astype(np.float32))
    ex = ex.reshape(N, 32, chunk)
    lsum = np.zeros((N, 32), np.float32)
    for k in range(chunk):
        lsum = lsum + ex[:, :, k]
    incl = lsum.copy()
    o = 1
    while o < 32:
        nxt = incl.copy()
        nxt[:, o:] = incl[:, o:] + incl[:, :-o]
        incl = nxt
        o <<= 1
    return ex, lsum, incl


def emulate_pick(logits, uni, rule="fixed"):
    """The kernels' inverse-CDF pick in float32, for rows ``logits`` (N, Q) and uniforms ``uni`` (N,);
    ``rule`` = "old" (excl = incl - lsum, no claim -> Q-1) or "fixed" (see the module docstring)."""
    lg = np.atleast_2d(np.asarray(logits, np.float32))
    N, Q = lg.shape
    chunk = (Q + 31) // 32
    ex, lsum, incl = _lane_sums(lg, chunk)
    total = incl[:, 31]
    target = (np.asarray(uni, np.float32).reshape(N) * total).astype(np.float32)
    if rule == "old":
        excl = incl - lsum
    elif rule == "fixed":
        excl = np.concatenate([np.zeros((N, 1), np.float32), incl[:, :31]], 1)
    else:
        raise ValueError(rule)
    t = target[:, None]
    claim = (t >= excl) & (t < incl)
    qidx = np.arange(32 * chunk).reshape(32, chunk)
    nz = ex > 0
    last_nz = np.where(nz, qidx[None], -1).max(2)                 # (N, 32): lane's last class with e > 0
    if rule == "old":
        cand = np.broadcast_to(np.minimum(qidx[:, -1], Q - 1), (N, 32)).copy()
    else:
        cand = np.maximum.accumulate(last_nz, axis=1)     # last class with e > 0 up to and including the lane
    found = np.zeros((N, 32), bool)
    c = incl - lsum                                   # both rules walk from incl - lsum
    for k in range(chunk):
        c = c + ex[:, :, k]
        hit = (c > t) & ~found & ((ex[:, :, k] > 0) if rule == "fixed" else True)
        cand[hit] = qidx[:, k][None].repeat(N, 0)[hit]
        found |= hit
    BIG = np.iinfo(np.int64).max
    pick = np.where(claim, cand, BIG).min(1)
    if rule == "old":
        return np.where(pick == BIG, Q - 1, pick)
    return np.where(pick == BIG, last_nz.max(1), pick)


def lane_boundaries(logits, chunk=None):
    """float32 emulated inclusive lane sums of lanes 0..30 (the 31 inner lane boundaries) and the total of a row."""
    lg = np.asarray(logits, np.float32)[None]
    chunk = chunk or (lg.shape[1] + 31) // 32
    _, _, incl = _lane_sums(lg, chunk)
    return incl[0, :31], incl[0, 31]


def boundary_uniforms(logits, ulps=8):
    """float32 uniforms whose uni * total lands within +-``ulps`` ulps of each of the 31 inner lane boundaries of the
    row, plus 0 and 1 - 2^-24."""
    bnd, total = lane_boundaries(logits)
    out = [np.float32(0.0), np.float32(1.0 - U24)]
    for bv in bnd:
        sp = np.spacing(np.float32(bv))
        for k in range(-ulps, ulps + 1):
            t = np.float32(bv) + np.float32(k) * sp
            u = np.float32(np.float64(t) / np.float64(total))
            if 0.0 <= u < 1.0:
                out.append(u)
    return np.unique(np.asarray(out, np.float32))


def gap_uniform(logits):
    """A float32 uniform whose target falls in a gap of the OLD rule (between lane l-1's incl and lane l's
    incl - lsum), or None when the row has no reachable gap."""
    lg = np.asarray(logits, np.float32)[None]
    _, lsum, incl = _lane_sums(lg, (lg.shape[1] + 31) // 32)
    incl, lsum = incl[0], lsum[0]
    total = incl[31]
    excl = incl - lsum
    for l in range(1, 32):
        lo, hi = incl[l - 1], excl[l]
        if not hi > lo:
            continue
        u0 = np.float32(np.float64(lo) / np.float64(total))
        for k in range(-4, 64):
            u = np.float32(u0 + np.float32(k) * np.spacing(u0))
            t = np.float32(u * total)
            if lo <= t < hi and 0 <= u < 1:
                return u
    return None
