# -*- coding: utf-8 -*-
"""GPU tier: every code path of the streaming kernels of csrc/elementwise.cu against float64, element by element.

The launchers pick a kernel from the shape, the table size and the pointer alignment.  Each case below computes which
one it takes from the launcher's own condition, prints it, and each test asserts that every branch was reached.

Exact results (the arithmetic is fixed, so the comparison is ``torch.equal``):
* ``wnb_front_embed_fwd``: out = bias + tap_0 + tap_1 + ... in tap order, each tap a table row (missing history adds
  nothing), restated in float32 in that order.
* ``wnb_aux_upsample_fwd``: haux[b][t U + j][a] = fmaf(h[b][a][t], w[j], bias) -- the correctly rounded h w + b -- and
  exactly 0 in the pad columns a >= A; U = 0 is the plain transpose.
* ``wnb_cross_entropy``: rows t < start get exactly 0 gradient.

Bounds (u = 2^-24, the fp32 unit roundoff; ``tc_reference.lin_bound(mag, K)`` = 4 K u mag):
* Sums (the embedding and up-sampling gradients).  Each output is init + a sum of n terms (the terms products h g
  formed by ``fmaf``, or plain dout values), evaluated as some tree of fp32 additions whose depth is at most the number
  of terms plus the number of partial sums (per-lane, per-warp, per-chunk or per-block slots) added afterwards, K.
  Any such evaluation is within gamma_K sum |terms| <= K u / (1 - K u) sum |terms| of the exact sum (Higham 3.1);
  lin_bound(sum |terms|, K) is four times that.  The final += into the caller's buffer adds u (|result| + |init|).
  For the embedding gradient K is taken as n_rows + 2048, which covers every partial-sum level of its three kernels
  (<= 512 lanes, one slot per SM, one reduction per token).  For the up-sampling gradient K is the depth of its own
  summation (derived at the check), far below the number of terms.  The bias of the up-sampling layer, a single scalar
  whose sum cancels heavily, is checked the same way: the bound is relative to sum |terms|, not to the result.
* Cross entropy, per row r with logits l (max m, s = sum_q expf(l_q - m), lse = m + logf(s)):  each expf is within
  2 ulp (2^-22 relative) of exp of its rounded argument, and the rounding of l_q - m (u |l_q - m|) changes exp(l_q - m)
  by at most that much relatively; x exp(-x) <= 1/e, so with s >= 1 the weighted sum of those is <= Q u / e, and the
  fp32 summation adds Q u: |s^ / s - 1| <= rel_s = 2^-22 + 1.4 Q u.  Then |lse^ - lse| <= rel_s + 2^-23 |log s| (logf,
  1 ulp) + u |lse| + slack, and the row loss lse - l_t adds u |lse - l_t|:
      e_row = 2^-22 + 1.5 Q u + 2^-22 |log s| + 2u (|lse| + |lse - l_t|)
  The loss is the double sum of the rows times inv_n = fl(1/n): |err| <= mean(e_row) + 2u |loss| (+ 1e-15 of the
  double sums).  The gradient p_q = expf(l_q - m) / s (times inv_n, minus 1/n at the target):
      e_dl = (1/n) (p (2^-22 + u |l_q - m| + rel_s + 4u) + u |p - [q = t]|) + 2u |dl| + 2^-146,
  the last term for gradients below the fp32 normal range (logits spread over +-1e3): there expf and the two products
  are exact only to within a few units of the smallest subnormal, 2^-149, each.

Determinism: the reducing kernels (``front_embed_bwd``, ``aux_upsample_bwd`` and the loss sum) are bit-identical over
repeated calls.  The largest err/bound of every case is printed.
"""
import math

import pytest
import torch

from tests import tc_reference as ref
from tests.test_gpu_tc_stages import Guarded

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F64 = torch.float64
ERR_INVALID = -1


def _lib():
    from pytorchwavenetvocoder_b200 import _lib as L
    return L, L.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _aligned(*ts):
    return all(t.data_ptr() % 16 == 0 for t in ts if t is not None)


def _misaligned(shape, fill=None):
    """a float32 tensor whose data starts one float past a 16-byte boundary"""
    n = int(math.prod(shape))
    buf = torch.empty(n + 4, device="cuda")
    v = buf[1:1 + n].view(*shape)
    if fill is not None:
        v.copy_(fill)
    v._keep = buf
    return v


def _sum_bound(mag, n_rows, got_init, want):
    """bound of init + (a sum with sum |terms| = mag), see the module docstring"""
    return ref.lin_bound(mag, n_rows + 2048) + U * (want.abs() + got_init.to(F64).abs())


class Branches:
    """records which kernel each case took; assert_all() checks every branch was reached"""

    def __init__(self, name, names):
        self.name, self.names, self.seen = name, set(names), set()

    def __call__(self, br, what):
        assert br in self.names, br
        self.seen.add(br)
        print("%s: %s -> %s" % (self.name, what, br))

    def assert_all(self):
        assert self.seen == self.names, "branches not reached: %s" % sorted(self.names - self.seen)


def _worst(name, got, want, bound):
    r = ref.assert_within(got, want, bound, name)
    print("largest err/bound [%s]: %.3g" % (name, r))
    return r


# ------------------------------------------------------------------------------------------------------------------
# front embedding
# ------------------------------------------------------------------------------------------------------------------
def _fe_fwd_branch(R, wf, bias, out):
    return "v4" if R % 4 == 0 and 256 % (R // 4) == 0 and _aligned(wf, bias, out) else "scalar"


def _fe_bwd_branch(R, Q, ks, dout):
    v4 = R % 4 == 0 and R // 4 <= 512 and _aligned(dout)
    if v4 and 256 % (R // 4) == 0 and ks * Q * R * 4 <= 160 * 1024:
        return "chunk"
    return "token<4>" if v4 else "token<1>"


def _tokens(x, Q):
    return x.remainder(Q)      # floor mod, as the kernels take x mod Q into [0, Q)


def _fe_reference(x, wf, bias, ks):
    """float32 restatement of the forward in kernel order: bias, then tap 0, 1, ... (tap k reads x[t - (ks-1-k)])"""
    B, T = x.shape
    Q = wf.shape[1]
    q = _tokens(x, Q)
    out = bias.expand(B, T, -1).clone()
    for k in range(ks):
        s_ = ks - 1 - k
        if s_ < T:
            out[:, s_:] = out[:, s_:] + wf[k][q[:, :T - s_]]
    return out


def _fe_bwd_reference(x, dout, Q, ks):
    """exact dwf (ks, Q, R) and dbias (R) sums and their sum |terms|, in float64"""
    B, T, R = dout.shape
    q = _tokens(x, Q)
    d64 = dout.to(F64)
    dwf = torch.zeros(ks, Q, R, dtype=F64, device="cuda")
    mag = torch.zeros_like(dwf)
    for k in range(ks):
        s_ = ks - 1 - k
        if s_ < T:
            idx = q[:, :T - s_].reshape(-1)
            dwf[k].index_add_(0, idx, d64[:, s_:].reshape(-1, R))
            mag[k].index_add_(0, idx, d64[:, s_:].abs().reshape(-1, R))
    return dwf, mag, d64.sum((0, 1)), d64.abs().sum((0, 1))


FE_CASES = [
    # R, Q, ks, B, T, misaligned
    (6, 256, 2, 2, 300, False),     # R % 4 != 0: scalar forward, scalar scan
    (64, 256, 2, 5, 301, False),    # chunked table (128 KB); 1505 rows in chunks of 12 that cross utterances
    (64, 256, 2, 1, 50, False),     # B T < SMs: most chunks empty
    (64, 256, 3, 2, 400, False),    # table 192 KB > 160 KB: per-token scan
    (64, 256, 4, 1, 3, False),      # T < ks
    (64, 256, 1, 2, 200, True),     # misaligned: scalar forward, scalar scan
    (96, 256, 1, 2, 130, False),    # R / 4 = 24 does not divide 256: scalar forward, per-token scan
    (128, 256, 2, 1, 2, False),     # table 256 KB: per-token; T < ks on one tap
    (512, 256, 2, 2, 257, False),   # the recipes' R: per-token scan
    (1024, 8, 1, 3, 40, False),     # R / 4 = 256: v4 forward, chunked table of 32 KB
    (1024, 256, 3, 1, 70, False),   # per-token scan with 2 lanes
    (2048, 33, 4, 2, 37, False),    # R / 4 = 512: scalar forward, per-token scan with one lane, ks = 4
]


def test_front_embed_every_branch():
    L_, lib = _lib()
    fwd = Branches("front_embed_fwd", ["v4", "scalar"])
    bwd = Branches("front_embed_bwd", ["chunk", "token<4>", "token<1>"])
    worst = 0.0
    for R, Q, ks, B, T, mis in FE_CASES:
        g = torch.Generator(device="cuda").manual_seed(R + Q + ks + B + T)
        what = "R=%d Q=%d ks=%d B=%d T=%d%s" % (R, Q, ks, B, T, " misaligned" if mis else "")
        x = torch.randint(-3 * Q, 3 * Q, (B, T), device="cuda", generator=g)     # tokens < 0 and >= Q
        wf = torch.randn(ks, Q, R, device="cuda", generator=g)
        bias = torch.randn(R, device="cuda", generator=g)
        G = Guarded()
        if mis:
            wf, bias = _misaligned(wf.shape, wf), _misaligned(bias.shape, bias)
            out = _misaligned((B, T, R), float("nan"))
        else:
            out = G((B, T, R))
        fwd(_fe_fwd_branch(R, wf, bias, out), what)
        L_.check(lib.wnb_front_embed_fwd(L_.ptr(x), L_.ptr(wf), L_.ptr(bias), L_.ptr(out), B, T, Q, R, ks,
                                         L_.stream()), "front_embed_fwd")
        torch.cuda.synchronize()
        G.check()
        want = _fe_reference(x, wf, bias, ks)
        assert torch.equal(out, want), "front_embed_fwd %s: max |diff| %g" % (what, (out - want).abs().max())
        # backward, three times from the same nonzero initial gradients: bit-identical
        dout = torch.randn(B, T, R, device="cuda", generator=g)
        if mis:
            dout = _misaligned(dout.shape, dout)
        bwd(_fe_bwd_branch(R, Q, ks, dout), what)
        init_w = torch.randn(ks, Q, R, device="cuda", generator=g)
        init_b = torch.randn(R, device="cuda", generator=g)
        runs = []
        for _ in range(3):
            G = Guarded()
            dwf, db = G(tuple(init_w.shape), init_w), G((R,), init_b)
            L_.check(lib.wnb_front_embed_bwd(L_.ptr(x), L_.ptr(dout), L_.ptr(dwf), L_.ptr(db), B, T, Q, R, ks,
                                             L_.stream()), "front_embed_bwd")
            torch.cuda.synchronize()
            G.check()
            runs.append((dwf.clone(), db.clone()))
        for dwf, db in runs[1:]:
            assert torch.equal(dwf, runs[0][0]) and torch.equal(db, runs[0][1]), "front_embed_bwd not reproducible"
        dwf, db = runs[0]
        s_w, m_w, s_b, m_b = _fe_bwd_reference(x, dout, Q, ks)
        want_w, want_b = init_w.to(F64) + s_w, init_b.to(F64) + s_b
        worst = max(worst, _worst("dwf " + what, dwf.reshape(ks * Q, R), want_w.reshape(ks * Q, R),
                                  _sum_bound(m_w, B * T, init_w, want_w).reshape(ks * Q, R)))
        worst = max(worst, _worst("dbias " + what, db, want_b, _sum_bound(m_b, B * T + Q, init_b, want_b)))
    fwd.assert_all()
    bwd.assert_all()
    print("front embed: largest err/bound %.3g" % worst)


def test_front_embed_bwd_rejects_before_launch():
    L_, lib = _lib()
    x = torch.zeros(1, 4, dtype=torch.int64, device="cuda")
    buf = torch.zeros(4 * 4 * 2050, device="cuda")
    for R, ks in [(2050, 1), (64, 5)]:
        n0 = L_.launch_count()
        rc = lib.wnb_front_embed_bwd(L_.ptr(x), L_.ptr(buf), L_.ptr(buf), L_.ptr(buf), 1, 4, 4, R, ks, L_.stream())
        assert rc == ERR_INVALID and L_.launch_count() == n0, (R, ks, rc)


# ------------------------------------------------------------------------------------------------------------------
# aux up-sampling
# ------------------------------------------------------------------------------------------------------------------
def _fmaf(h, w, b):
    """correctly rounded float32 h w + b (h, w, b float32, broadcast): the float64 sum of the exact product, rounded to
    float32, is wrong only when it lands exactly halfway between two floats; the exact remainder (TwoSum) then says which
    way the true value lies"""
    p = h.to(F64) * w.to(F64)                        # exact (24 + 24 bits)
    b64 = b.to(F64).expand_as(p)
    s = p + b64
    bv = s - p
    e = (p - (s - bv)) + (b64 - bv)                  # s + e == p + b exactly
    r = s.to(torch.float32)
    r64 = r.to(F64)
    toward = torch.where(s > r64, torch.full_like(r, float("inf")), torch.full_like(r, -float("inf")))
    n = torch.nextafter(r, toward)
    half = (s != r64) & (s == (r64 + n.to(F64)) / 2)
    # at a tie s rounds to even; the exact value p + b = s + e lies beyond s (away from r) iff e has the sign of s - r
    away = half & (e != 0) & ((e > 0) == (s > r64))
    return torch.where(away, n, r)


def _up_fwd_branch(Ap, haux):
    return "v4" if Ap % 4 == 0 and _aligned(haux) else "scalar"


UP_FWD_CASES = [
    # B, A, Ap, Tf, U, misaligned
    (2, 29, 32, 5, 0, False),       # plain transpose
    (1, 1, 4, 1, 1, False),         # Tf = 1, A = 1
    (3, 33, 35, 7, 80, False),      # Ap % 4 != 0: scalar
    (2, 256, 260, 3, 128, False),
    (1, 29, 32, 600, 129, False),   # B Tf above 4 SMs
    (4, 33, 64, 2, 256, True),      # misaligned output: scalar
    (1, 256, 257, 1, 0, False),     # transpose, scalar, Tf = 1
]


def test_aux_upsample_fwd_every_branch():
    L_, lib = _lib()
    br = Branches("aux_upsample_fwd", ["v4", "scalar"])
    for B, A, Ap, Tf, Uf, mis in UP_FWD_CASES:
        g = torch.Generator(device="cuda").manual_seed(B + A + Ap + Tf + Uf)
        what = "B=%d A=%d Ap=%d Tf=%d U=%d%s" % (B, A, Ap, Tf, Uf, " misaligned" if mis else "")
        h = torch.randn(B, A, Tf, device="cuda", generator=g)
        w = torch.randn(max(Uf, 1), device="cuda", generator=g)
        bias = torch.randn(1, device="cuda", generator=g)
        T = Tf * Uf if Uf else Tf
        G = Guarded()
        haux = _misaligned((B, T, Ap), float("nan")) if mis else G((B, T, Ap))
        br(_up_fwd_branch(Ap, haux), what)
        L_.check(lib.wnb_aux_upsample_fwd(L_.ptr(h), L_.ptr(w) if Uf else None, L_.ptr(bias) if Uf else None,
                                          L_.ptr(haux), B, A, Ap, Tf, Uf, L_.stream()), "aux_upsample_fwd")
        torch.cuda.synchronize()
        G.check()
        assert torch.all(haux[:, :, A:] == 0), what     # pad columns exactly 0 (+0 or -0 both compare equal)
        ht = h.transpose(1, 2)                            # (B, Tf, A)
        if Uf:
            want = _fmaf(ht[:, :, None, :], w[None, None, :, None], bias).reshape(B, T, A)
        else:
            want = ht
        assert torch.equal(haux[:, :, :A], want), "%s: max |diff| %g" % (what, (haux[:, :, :A] - want).abs().max())
    br.assert_all()


UP_BWD_CASES = [
    # B, A, Ap, Tf, U
    (1, 1, 32, 1, 1),
    (2, 29, 32, 9, 80),
    (3, 33, 64, 5, 128),
    (1, 256, 256, 700, 129),   # B Tf above 4 SMs: blocks loop over items
    (2, 29, 32, 40, 256),      # two j passes
    (5, 256, 260, 3, 256),
]


def test_aux_upsample_bwd():
    L_, lib = _lib()
    sms = _sms()
    below = above = False
    worst = 0.0
    for B, A, Ap, Tf, Uf in UP_BWD_CASES:
        g = torch.Generator(device="cuda").manual_seed(B + A + Ap + Tf + Uf)
        what = "B=%d A=%d Ap=%d Tf=%d U=%d" % (B, A, Ap, Tf, Uf)
        below |= B * Tf < 4 * sms
        above |= B * Tf > 4 * sms
        T = Tf * Uf
        h = torch.randn(B, A, Tf, device="cuda", generator=g)
        dh = torch.randn(B, T, Ap, device="cuda", generator=g)
        dh[:, :, A:] = 1e6                 # pad columns carry no gradient: a read of them would show
        init_w = torch.randn(Uf, device="cuda", generator=g)
        init_b = torch.randn(1, device="cuda", generator=g)
        runs = []
        for _ in range(3):
            G = Guarded()
            dw, db = G((Uf,), init_w), G((1,), init_b)
            L_.check(lib.wnb_aux_upsample_bwd(L_.ptr(h), L_.ptr(dh), L_.ptr(dw), L_.ptr(db), B, A, Ap, Tf, Uf,
                                              L_.stream()), "aux_upsample_bwd")
            torch.cuda.synchronize()
            G.check()
            runs.append((dw.clone(), db.clone()))
        for dw, db in runs[1:]:
            assert torch.equal(dw, runs[0][0]) and torch.equal(db, runs[0][1]), "aux_upsample_bwd not reproducible"
        dw, db = runs[0]
        d64 = dh[:, :, :A].to(F64).reshape(B, Tf, Uf, A)
        h64 = h.to(F64).transpose(1, 2)[:, :, None, :]        # (B, Tf, 1, A)
        want_w = init_w.to(F64) + (d64 * h64).sum((0, 1, 3))
        mag_w = (d64 * h64).abs().sum((0, 1, 3))
        want_b = init_b.to(F64) + d64.sum()
        mag_b = d64.abs().sum().reshape(1)
        # summation depth of aux_upsample_bwd_kernel: a lane's fmaf chain over its block's (b, tf) items and 8 channels,
        # the 5-step warp sum, then the per-block slots in order and the += (dbias: a lane's running sum over every j
        # of its warp, the warp sum, the 8 warps, the slots)
        grid = min(B * Tf, 4 * sms)
        per = -(-(B * Tf) // grid)
        k_w = per * 8 + 5 + grid + 1
        k_b = per * 8 * -(-Uf // 8) + 5 + 8 + grid + 1
        worst = max(worst, _worst("dw " + what, dw.reshape(1, -1), want_w.reshape(1, -1),
                                  ref.lin_bound(mag_w, k_w).reshape(1, -1)
                                  + U * (want_w.abs() + init_w.to(F64).abs()).reshape(1, -1)))
        worst = max(worst, _worst("dbias " + what, db, want_b,
                                  ref.lin_bound(mag_b, k_b) + U * (want_b.abs() + init_b.to(F64).abs())))
    assert below and above
    print("aux up-sampling backward: largest err/bound %.3g" % worst)


def test_aux_upsample_bwd_rejects_a257():
    L_, lib = _lib()
    buf = torch.zeros(2 * 260 * 4, device="cuda")
    n0 = L_.launch_count()
    rc = lib.wnb_aux_upsample_bwd(L_.ptr(buf), L_.ptr(buf), L_.ptr(buf), L_.ptr(buf), 1, 257, 260, 1, 2, L_.stream())
    assert rc == ERR_INVALID and L_.launch_count() == n0, rc


# ------------------------------------------------------------------------------------------------------------------
# cross entropy
# ------------------------------------------------------------------------------------------------------------------
def _ce_branch(Q, logits, dlogits):
    return "q256" if Q == 256 and _aligned(logits, dlogits) else "general"


def _ce_reference(logits, target, start):
    """float64 loss, dlogits and their bounds (module docstring)"""
    B, T, Q = logits.shape
    l64 = logits.to(F64)
    n = B * (T - start)
    m = l64.max(-1, keepdim=True).values
    s = torch.exp(l64 - m).sum(-1, keepdim=True)
    lse = m + torch.log(s)
    lt = l64.gather(-1, target[..., None])
    row = (lse - lt)[..., 0]
    rel_s = 2.0 ** -22 + 1.4 * Q * U
    e_row = 2.0 ** -22 + 1.5 * Q * U + 2.0 ** -22 * torch.log(s)[..., 0].abs() + 2 * U * (lse[..., 0].abs() + row.abs())
    loss = row[:, start:].sum() / n
    e_loss = e_row[:, start:].sum() / n + 2 * U * loss.abs() + 1e-15 * row[:, start:].abs().sum() / n
    p = torch.exp(l64 - lse)
    onehot = torch.zeros_like(p).scatter_(-1, target[..., None], 1.0)
    dl = (p - onehot) / n
    e_dl = ((p * (2.0 ** -22 + U * (l64 - m).abs() + rel_s + 4 * U) + U * (p - onehot).abs()) / n + 2 * U * dl.abs()
            + 2.0 ** -146)
    dl[:, :start] = 0
    e_dl[:, :start] = 0
    return loss, e_loss, dl, e_dl


CE_CASES = [
    # B, T, Q, start, spread, form: "out" (separate dlogits), "none" (dlogits NULL), "alias" (in place), "mis"
    (2, 100, 256, 0, 3.0, "out"),
    (3, 70, 256, 69, 1e3, "out"),     # start = T - 1, logits over +-1e3
    (2, 50, 256, 7, 3.0, "none"),
    (1, 2000, 256, 11, 30.0, "alias"),
    (2, 40, 256, 3, 3.0, "mis"),      # Q = 256 misaligned: the general kernel
    (4, 33, 2, 0, 3.0, "out"),
    (2, 65, 33, 64, 1e3, "alias"),
    (1, 129, 1000, 5, 10.0, "out"),
]


def test_cross_entropy_every_branch():
    L_, lib = _lib()
    br = Branches("cross_entropy", ["q256", "general"])
    worst = 0.0
    for B, T, Q, start, spread, form in CE_CASES:
        g = torch.Generator(device="cuda").manual_seed(B + T + Q + start)
        what = "B=%d T=%d Q=%d start=%d spread=%g %s" % (B, T, Q, start, spread, form)
        lg = (torch.rand(B, T, Q, device="cuda", generator=g) * 2 - 1) * spread
        target = torch.randint(0, Q, (B, T), device="cuda", generator=g)
        want_loss, e_loss, want_dl, e_dl = _ce_reference(lg, target, start)
        G = Guarded()
        if form == "mis":
            logits = _misaligned(lg.shape, lg)
            dl = _misaligned(lg.shape, float("nan"))
        else:
            logits = G(tuple(lg.shape), lg)
            dl = {"out": G(tuple(lg.shape)), "none": None, "alias": logits}[form]
        br(_ce_branch(Q, logits, dl), what)
        loss0 = 0.75
        losses = []
        for _ in range(1 if form == "alias" else 3):
            loss_sum = torch.full((1,), loss0, dtype=F64, device="cuda")
            L_.check(lib.wnb_cross_entropy(L_.ptr(logits), L_.ptr(target), L_.ptr(loss_sum), L_.ptr(dl), B, T, Q,
                                           start, L_.stream()), "cross_entropy")
            torch.cuda.synchronize()
            losses.append(loss_sum.clone())
        G.check()
        for ls in losses[1:]:
            assert torch.equal(ls, losses[0]), "loss sum not reproducible"
        worst = max(worst, _worst("loss " + what, losses[0] - loss0, want_loss.reshape(1), e_loss.reshape(1)))
        if dl is not None:
            assert torch.equal(dl[:, :start], torch.zeros_like(dl[:, :start])), "rows t < start: exactly 0"
            worst = max(worst, _worst("dlogits " + what, dl, want_dl, e_dl))
        else:
            assert torch.equal(logits, lg), "dlogits = NULL must leave the logits alone"
    br.assert_all()
    print("cross entropy: largest err/bound %.3g" % worst)


@pytest.mark.parametrize("Q", [256, 33])
def test_cross_entropy_out_of_range_target_is_nan(Q):
    L_, lib = _lib()
    B, T = 1, 8
    logits = torch.randn(B, T, Q, device="cuda")
    for bad in (-1, Q):
        target = torch.zeros(B, T, dtype=torch.int64, device="cuda")
        target[0, 5] = bad
        loss_sum = torch.zeros(1, dtype=F64, device="cuda")
        dl = torch.empty_like(logits)
        L_.check(lib.wnb_cross_entropy(L_.ptr(logits), L_.ptr(target), L_.ptr(loss_sum), L_.ptr(dl), B, T, Q, 0,
                                       L_.stream()), "cross_entropy")
        torch.cuda.synchronize()
        assert torch.isnan(loss_sum).all(), (Q, bad)
