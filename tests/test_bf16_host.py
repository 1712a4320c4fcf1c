# -*- coding: utf-8 -*-
"""CPU tier: the bf16 operand path (math_mode="bf16") without a GPU.

* ``to_bf16`` -- the operand conversion the GPU tests hand to tests/tc_reference.py as ``cv=`` -- is round to nearest
  even, checked against a bit-level implementation on ties, carries into the exponent, the largest finite value and
  subnormals.
* A float32 emulation of the kernels' bf16 arithmetic (bf16 operands, exact products, fp32 accumulation per k16 MMA)
  stays within tc_reference's bounds when they are computed with ``cv=to_bf16``.
* The host logic of the C ABI: which shapes the bf16 path covers, and that unknown math modes are refused.
"""
import numpy as np
import pytest
import torch

from tests import tc_reference as ref
from tests.test_tc_reference import Emu


def to_bf16(x):
    """fp32 tensor -> float64 tensor of the bf16 value (round to nearest even) the tensor cores multiply with."""
    return x.detach().to(torch.float32).to(torch.bfloat16).to(torch.float64)


def _bf16_rne_bits(f32):
    """bit-level round to nearest even of fp32 values (no NaN) to bf16, as fp32 bit patterns"""
    b = np.asarray(f32, dtype=np.float32).view(np.uint32).astype(np.uint64)
    lsb = (b >> 16) & 1
    return (((b + 0x7FFF + lsb) >> 16) << 16).astype(np.uint32)


def _check(vals):
    v = np.asarray(vals, dtype=np.float32)
    got = to_bf16(torch.from_numpy(v)).to(torch.float32).numpy().view(np.uint32)
    want = _bf16_rne_bits(v)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(float(v[i]), hex(int(got[i])), hex(int(want[i]))) for i in bad[:5]]
    return got.view(np.float32)


def test_to_bf16_is_round_to_nearest_even():
    one = 1.0
    u = 2.0 ** -7                                                 # bf16 ulp at 1
    got = _check([one + u / 2, one + 3 * u / 2, -(one + u / 2), one + u / 2 + 2.0 ** -20, one + 0.75 * u])
    assert list(got) == [1.0, one + 2 * u, -1.0, one + u, one + u]   # ties to even, above the tie rounds up
    # carries into the exponent: the largest fp32 below 2, and the largest fp32 below 2^k for several k
    below = np.nextafter(np.float32([2.0, 4.0, 1024.0, 2.0 ** -100]), np.float32(0))
    assert list(_check(below)) == [2.0, 4.0, 1024.0, 2.0 ** -100]
    # the largest finite fp32 rounds to infinity; the largest finite bf16 is kept
    fmax = np.finfo(np.float32).max
    bmax = np.uint32(0x7F7F0000).view(np.float32)
    got = _check([fmax, -fmax, bmax])
    assert np.isinf(got[0]) and got[0] > 0 and np.isinf(got[1]) and got[1] < 0 and got[2] == bmax
    # subnormals: rounded, not flushed; the smallest ones round to zero or to the smallest bf16 subnormal
    sub = np.array([0x00010000, 0x00018000, 0x00028000, 0x00008000, 0x00008001, 0x007FFFFF, 0x80018000],
                   dtype=np.uint32).view(np.float32)
    got = _check(sub).view(np.uint32)
    assert list(got) == [0x00010000, 0x00020000, 0x00020000, 0x00000000, 0x00010000, 0x00800000, 0x80020000]
    # a broad sample of finite bit patterns
    rng = np.random.RandomState(0)
    bits = rng.randint(0, 2 ** 32, size=200000, dtype=np.uint64).astype(np.uint32)
    vals = bits.view(np.float32)
    _check(vals[np.isfinite(vals)])


class EmuBf16(Emu):
    """bf16 operands, exact products, fp32 accumulation over a shuffled K in chunks of 16 (the per-k16 MMA) summed in
    fp32 in shuffled order; tanh.approx as tanh * (1 + delta), |delta| <= 2^-11"""

    def mm(self, a, w):
        A = to_bf16(a.float()).reshape(-1, a.shape[-1])
        Wt = to_bf16(w.float())
        P = (A[:, None, :] * Wt[None, :, :]).float()          # exact: 8 x 8 significant bits
        K = P.shape[-1]
        P = P[..., torch.randperm(K, generator=self.g)]
        chunks = []
        for c0 in range(0, K, 16):
            acc = torch.zeros(P.shape[:2], dtype=torch.float32)
            for k in range(c0, min(K, c0 + 16)):
                acc = acc + P[..., k]
            chunks.append(acc)
        acc = torch.zeros(P.shape[:2], dtype=torch.float32)
        for i in torch.randperm(len(chunks), generator=self.g).tolist():
            acc = acc + chunks[i]
        return acc.reshape(*a.shape[:-1], w.shape[0])


def _rand(g, *sh, scale=1.0):
    return torch.randn(*sh, generator=g, dtype=torch.float32) * scale


@pytest.mark.parametrize("seed", range(12))
def test_bounds_hold_under_emulated_bf16_arithmetic(seed):
    """The stages of one composed block and its weight gradient, bounds from tc_reference with cv=to_bf16."""
    g = torch.Generator().manual_seed(100 + seed)
    em = EmuBf16(seed)
    R, Ap, ks = 64, 32, [1, 2, 3][seed % 3]
    B, T, d, S = 2, [1, 13, 40][seed % 3], 1 + seed % 7, 96
    K1 = ks * R + Ap
    cv = to_bf16
    xin, haux = _rand(g, B, T, R), _rand(g, B, T, Ap)
    w1, b1 = _rand(g, 2 * R, K1, scale=K1 ** -0.5), _rand(g, 2 * R, scale=0.3)
    w2, b2 = _rand(g, R + S, R, scale=R ** -0.5), _rand(g, R + S, scale=0.1)
    worst = 0.0
    s, th = em.gates(em.pre(xin, haux, w1, b1, d, ks))
    z = s * th
    worst = max(worst, ref.assert_within(z, *ref.gate_fwd(xin, haux, w1, b1, d, ks, cv=cv), "z"))
    xout = em.mm(z, w2[:R]) + b2[:R] + xin
    worst = max(worst, ref.assert_within(xout, *ref.res_out(xin, z, w2[:R], b2[:R], cv=cv), "xout"))
    sk = em.mm(z, w2[R:]) + b2[R:]
    worst = max(worst, ref.assert_within(sk, *ref.skip_gemm(z, w2[R:], b2[R:], False, cv=cv), "skip"))
    dskip, dout = _rand(g, B, T, S), _rand(g, B, T, R)
    dz = em.mm(torch.cat([dout, dskip], -1), w2.t().contiguous())
    dz_ref, e_dz = ref.dz_perblock(dout, dskip, w2, cv=cv)
    worst = max(worst, ref.assert_within(dz, dz_ref, e_dz, "dz"))
    dpre = torch.cat([dz * th * s * (1 - s), dz * s * (1 - th * th)], -1)
    worst = max(worst, ref.assert_within(dpre, *ref.gate_bwd(xin, haux, w1, b1, d, ks, dz_ref, e_dz, cv=cv), "dpre"))
    dx = sum(em.mm(ref.tshift(dpre, (ks - 1 - j) * d), w1[:, j * R:(j + 1) * R].t().contiguous())
             for j in range(ks)) + dout
    worst = max(worst, ref.assert_within(dx, *ref.dx_stage(dpre, w1, d, ks, dout, cv=cv), "dx"))
    bm = torch.cat(ref.taps(xin, ks, d) + [haux], -1)
    init = _rand(g, 2 * R, K1)
    dw1 = em.mm(dpre.reshape(-1, 2 * R).t().contiguous(), bm.reshape(-1, K1).t().contiguous()) + init
    (dw, bw), _ = ref.wgrad(dpre, ref.taps(xin, ks, d) + [haux], init, cv=cv)
    worst = max(worst, ref.assert_within(dw1, dw, bw, "dW1"))
    print("seed %d: largest err/bound %.3f" % (seed, worst))


def test_tf32_bounds_do_not_cover_bf16_operands():
    """The bound is specific to the conversion: a bf16 result checked with the tf32 conversion fails (so cv= matters)."""
    g = torch.Generator().manual_seed(7)
    a, w = _rand(g, 4, 64, 256), _rand(g, 128, 256, scale=1 / 16)
    got = EmuBf16(0).mm(a, w)
    ref.assert_within(got, *ref.skip_gemm(a, w, None, False, cv=to_bf16), "bf16")
    with pytest.raises(AssertionError):
        ref.assert_within(got, *ref.skip_gemm(a, w, None, False, cv=ref.to_tf32), "bf16 vs tf32 bound")


def test_abi_bf16_host_logic_without_gpu():
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    BF16, TF32, FP32 = _lib.MATH_BF16, _lib.MATH_TF32, _lib.MATH_FP32
    assert BF16 == 2
    sup = lib.wnb_resblock_fwd_supported
    assert sup(512, 256, 96, 3, BF16) == 2            # ljspeech recipe shape: composed path
    assert sup(512, 256, 32, 2, BF16) == 2            # arctic recipe shape
    assert sup(64, 512, 32, 2, BF16) == 2             # BASELINE shape: composed in bf16 (the fused kernel is tf32)
    assert sup(64, 512, 32, 2, TF32) == 1
    assert sup(96, 256, 32, 2, BF16) == 0             # R not a multiple of 64
    assert sup(512, 384, 32, 2, BF16) == 0            # S outside the GEMM's N list
    assert sup(512, 256, 32, 4, BF16) == 0            # kernel_size 4
    assert sup(64, 512, 32, 2, 7) == 0                # unknown math mode
    assert sup(64, 512, 32, 2, FP32) == 1
    for L in (1, 30):
        assert lib.wnb_stack_supported(64, 512, 32, 2, L, BF16) == 0
        assert lib.wnb_stack_supported(512, 256, 96, 3, L, BF16) == 0
    fake = 256   # never dereferenced: every call below is refused before any CUDA work
    rc = lib.wnb_resblock_fwd(*[fake] * 9, 2, 64, 96, 256, 32, 2, 1, 1, BF16, None)
    assert rc == -1 and b"not supported by the bf16" in lib.wnb_last_error()
    rc = lib.wnb_resblock_fwd(*[fake] * 9, 2, 64, 512, 256, 32, 2, 1, 1, 7, None)
    assert rc == -1 and b"unknown math_mode 7" in lib.wnb_last_error()
    rc = lib.wnb_resblock_bwd(*[fake] * 15, 2, 64, 96, 256, 32, 2, 1, BF16, None)
    assert rc == -1 and b"not supported by the bf16" in lib.wnb_last_error()
    rc = lib.wnb_resblock_bwd(*[fake] * 15, 2, 64, 512, 256, 32, 2, 1, 7, None)
    assert rc == -1 and b"unknown math_mode 7" in lib.wnb_last_error()
    rc = lib.wnb_post_fwd(*[fake] * 7, 2, 64, 384, 256, BF16, 0, None)
    assert rc == -1 and b"not supported by the bf16" in lib.wnb_last_error()
    rc = lib.wnb_post_fwd(*[fake] * 7, 2, 64, 256, 256, 9, 0, None)
    assert rc == -1 and b"unknown math_mode 9" in lib.wnb_last_error()
    rc = lib.wnb_post_bwd(*[fake] * 11, 2, 64, 256, 256, 9, None)
    assert rc == -1 and b"unknown math_mode 9" in lib.wnb_last_error()


def test_model_math_mode_host_logic():
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import WaveNet
    from pytorchwavenetvocoder_b200.nets.wavenet import bf16_supported
    net = WaveNet(256, 28, 64, 128, 3, 1, 2, 0)
    net.math_mode = "bf16"
    assert net._math() == _lib.MATH_BF16
    net.math_mode = "fp16"
    with pytest.raises(ValueError, match="fp32, tf32 or bf16"):
        net._math()
    assert bf16_supported((256, 80, 512, 256, 10, 3, 3, 256))
    assert bf16_supported((256, 28, 512, 256, 10, 3, 2, 80))
    assert bf16_supported((256, 28, 64, 512, 10, 3, 2, 80))
    assert not bf16_supported((256, 28, 96, 256, 10, 3, 2, 80))
    assert not bf16_supported((256, 28, 512, 384, 10, 3, 2, 80))
    assert not bf16_supported((200, 28, 512, 256, 10, 3, 2, 80))
