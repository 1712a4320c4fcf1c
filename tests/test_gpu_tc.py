# -*- coding: utf-8 -*-
"""GPU tier: the wgmma/TMA tensor-core residual-block paths (math_mode="tf32") against the fp32 FFMA kernel
and the fp64 oracle.

Stated tolerance for the tf32 path (tf32 multiplies = 10-bit mantissa operands, fp32 accumulate,
tanh.approx gate):  single block |err| <= 4e-3 * max|ref|;  30-layer logits |err| <= 5e-2 abs with
argmax agreement >= 97 % where the oracle's top-2 margin exceeds 0.1.
"""
import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu


def _block(mode, xin, haux, W1, b1, W2, b2, d, skip0, last):
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    B, T, R = xin.shape
    S = W2.shape[0] - R
    xout = None if last else torch.full_like(xin, float("nan"))
    skip = torch.zeros(B, T, S, device="cuda") if skip0 is None else skip0.clone()
    _lib.check(lib.wnb_resblock_fwd(_lib.ptr(xin), _lib.ptr(haux), _lib.ptr(W1), _lib.ptr(b1), _lib.ptr(W2),
                                    _lib.ptr(b2), _lib.ptr(xout), _lib.ptr(skip), None, B, T, R, S, 32, 2, d,
                                    1 if skip0 is None else 0, mode, _lib.stream()), "resblock_fwd")
    torch.cuda.synchronize()
    return xout, skip


@pytest.mark.parametrize("d,T,last,init", [(1, 256, False, True), (4, 384, False, False), (512, 1024, False, False),
                                            (2, 200, False, False), (64, 128, True, False), (128, 23040, False, True)])
def test_single_block_tf32_vs_fp32(d, T, last, init):
    from pytorchwavenetvocoder_b200 import _lib
    torch.manual_seed(d + T)
    B, R, S, Ap = 2, 64, 512, 32
    xin = torch.randn(B, T, R, device="cuda")
    haux = torch.randn(B, T, Ap, device="cuda")
    haux[:, :, 28:] = 0
    K1 = 2 * R + Ap
    W1 = (torch.randn(2 * R, K1, device="cuda") / np.sqrt(K1)).contiguous()
    W2 = (torch.randn(R + S, R, device="cuda") / np.sqrt(R)).contiguous()
    b1 = 0.1 * torch.randn(2 * R, device="cuda")
    b2 = 0.1 * torch.randn(R + S, device="cuda")
    skip0 = None if init else torch.randn(B, T, S, device="cuda")
    xo_ref, sk_ref = _block(_lib.MATH_FP32, xin, haux, W1, b1, W2, b2, d, skip0, last)
    xo, sk = _block(_lib.MATH_TF32, xin, haux, W1, b1, W2, b2, d, skip0, last)
    tol = 4e-3
    assert torch.isfinite(sk).all()
    err_s = (sk - sk_ref).abs().max().item() / sk_ref.abs().max().item()
    assert err_s < tol, ("skip", err_s)
    if not last:
        assert torch.isfinite(xo).all()
        err_x = (xo - xo_ref).abs().max().item() / xo_ref.abs().max().item()
        assert err_x < tol, ("xout", err_x)


def test_full_forward_tf32_vs_oracle():
    cfg = O.Config(256, 28, 64, 512, 10, 3, 2, 80)
    p = O.make_params(cfg, 3)
    net = our_model(cfg, p, math_mode="tf32").eval()
    rng = np.random.RandomState(4)
    B, T = 2, 1600
    x = rng.randint(0, 256, size=(B, T)).astype(np.int64)
    h = rng.standard_normal((B, 28, T // 80)).astype(np.float32)
    with torch.no_grad():
        y = net(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda()).cpu().numpy()
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    ref = O.forward(cfg, p64, x, h.astype(np.float64))
    err = np.abs(y - ref).max()
    assert err < 5e-2, err
    srt = np.sort(ref, axis=-1)
    clear = (srt[..., -1] - srt[..., -2]) > 0.1
    agree = (y.argmax(-1) == ref.argmax(-1))[clear].mean()
    assert agree >= 0.97, agree


def test_training_step_tf32_close_to_fp32():
    """forward in tf32 + backward: loss within 1e-3 and every gradient tensor within 5 % (relative
    Frobenius norm) of the all-fp32 run."""
    from pytorchwavenetvocoder_b200.nets import cross_entropy
    cfg = O.Config(256, 28, 64, 128, 6, 2, 2, 16)
    p = O.make_params(cfg, 8)
    rng = np.random.RandomState(2)
    B, T = 2, 512
    x = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    t = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    h = torch.from_numpy(rng.standard_normal((B, 28, T // 16)).astype(np.float32)).cuda()
    res = {}
    for mode in ("fp32", "tf32"):
        net = our_model(cfg, p, math_mode=mode).train()
        loss = cross_entropy(net(x, h), t, 64)
        loss.backward()
        res[mode] = (loss.item(), {k: v.grad.clone() for k, v in net.named_parameters() if v.grad is not None})
    assert abs(res["fp32"][0] - res["tf32"][0]) < 1e-3
    for k, g in res["fp32"][1].items():
        g2 = res["tf32"][1][k]
        if g.numel() == 1:      # scalar sums with heavy cancellation (upsampling bias): absolute bound
            assert (g - g2).abs().item() <= 3e-3, k
        else:
            tol = 0.10 if g.dim() == 1 else 0.05     # bias gradients are small sums with cancellation
            assert (g - g2).norm().item() <= tol * g.norm().item() + 1e-7, k


def test_block_backward_tf32_vs_fp32_single_layer():
    """wnb_resblock_bwd in tf32 mode (tensor-core weight gradients) vs the all-FFMA path, one block."""
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    torch.manual_seed(5)
    B, T, R, S, Ap, d = 2, 1000, 64, 512, 32, 4
    K1 = 2 * R + Ap
    xin = torch.randn(B, T, R, device="cuda")
    haux = torch.randn(B, T, Ap, device="cuda"); haux[:, :, 28:] = 0
    dout = torch.randn(B, T, R, device="cuda")
    dskip = torch.randn(B, T, S, device="cuda")
    W1 = (torch.randn(2 * R, K1, device="cuda") / np.sqrt(K1)).contiguous()
    W2 = (torch.randn(R + S, R, device="cuda") / np.sqrt(R)).contiguous()
    b1 = 0.1 * torch.randn(2 * R, device="cuda")
    w1t, w2t = W1.t().contiguous(), W2.t().contiguous()
    ws = torch.empty(lib.wnb_resblock_bwd_workspace(B, T, R, S, Ap, 2) // 4, device="cuda")
    out = {}
    for mode in (_lib.MATH_FP32, _lib.MATH_TF32):
        dx = torch.empty(B, T, R, device="cuda")
        dh = torch.zeros(B, T, Ap, device="cuda")
        dw1, db1 = torch.zeros(2 * R, K1, device="cuda"), torch.zeros(2 * R, device="cuda")
        dw2, db2 = torch.zeros(R + S, R, device="cuda"), torch.zeros(R + S, device="cuda")
        _lib.check(lib.wnb_resblock_bwd(_lib.ptr(xin), _lib.ptr(haux), _lib.ptr(dout), _lib.ptr(dskip), _lib.ptr(W1),
                                        _lib.ptr(b1), _lib.ptr(w1t), _lib.ptr(w2t), _lib.ptr(dx), _lib.ptr(dh),
                                        _lib.ptr(dw1), _lib.ptr(db1), _lib.ptr(dw2), _lib.ptr(db2), _lib.ptr(ws),
                                        B, T, R, S, Ap, 2, d, mode, _lib.stream()), "resblock_bwd")
        torch.cuda.synchronize()
        out[mode] = dict(dx=dx, dh=dh, dw1=dw1, db1=db1, dw2=dw2, db2=db2)
    for k, ref in out[_lib.MATH_FP32].items():
        got = out[_lib.MATH_TF32][k]
        rel = (got - ref).norm().item() / ref.norm().item()
        assert rel < 5e-3, (k, rel)


def test_tf32_training_learns():
    """System-level sanity of the whole tf32 training path (fwd + fused CE + tensor-core bwd + Adam): fitting one
    fixed batch of a mu-law sine must bring the loss well below its initial value (ln 256 = 5.55)."""
    from pytorchwavenetvocoder_b200.nets import WaveNet, cross_entropy, initialize
    torch.manual_seed(0)
    net = WaveNet(256, 28, 64, 128, 6, 2, 2, 16).cuda()
    net.apply(initialize)
    net.math_mode = "tf32"
    net.train()
    opt = torch.optim.Adam(net.parameters(), lr=2e-3)
    T, B = 1024, 4
    tt = np.arange(T + 1) / 16000.0
    wav = np.stack([0.5 * np.sin(2 * np.pi * (200 + 40 * b) * tt) for b in range(B)])
    q = O.encode_mu_law(wav, 256)
    x = torch.from_numpy(q[:, :-1]).cuda()
    t = torch.from_numpy(q[:, 1:]).cuda()
    h = torch.randn(B, 28, T // 16, device="cuda")
    rf = net.receptive_field
    losses = []
    for _ in range(60):
        loss = cross_entropy(net(x, h), t, rf)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all()
    assert losses[0] > 5.0 and losses[-1] < 0.6 * losses[0], (losses[0], losses[-1])


# ------------------------------------------------------------------------------------------------------------
# composed tensor-core path: shapes outside the fused kernel (e.g. the recipes' 512 res / 256 skip, kernel_size 3)
# ------------------------------------------------------------------------------------------------------------
def _block_general(mode, R, S, Ap, ks, d, B, T, last, init, seed):
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)  # noqa: E731
    K1 = ks * R + Ap
    xin, haux = rn(B, T, R), rn(B, T, Ap)
    W1 = (rn(2 * R, K1) / np.sqrt(K1)).contiguous()
    W2 = (rn(R + S, R) / np.sqrt(R)).contiguous()
    b1, b2 = 0.1 * rn(2 * R), 0.1 * rn(R + S)
    skip = torch.zeros(B, T, S, device="cuda") if init else rn(B, T, S)
    xout = None if last else torch.full((B, T, R), float("nan"), device="cuda")
    zbuf = torch.empty(B, T, R, device="cuda") if lib.wnb_resblock_fwd_supported(R, S, Ap, ks, mode) == 2 else None
    _lib.check(lib.wnb_resblock_fwd(_lib.ptr(xin), _lib.ptr(haux), _lib.ptr(W1), _lib.ptr(b1), _lib.ptr(W2),
                                    _lib.ptr(b2), _lib.ptr(xout), _lib.ptr(skip), _lib.ptr(zbuf), B, T, R, S, Ap, ks, d,
                                    1 if init else 0, mode, _lib.stream()), "resblock_fwd")
    # backward with the same operands
    dout = None if last else rn(B, T, R)
    dskip = rn(B, T, S)
    w1t, w2t = W1.t().contiguous(), W2.t().contiguous()
    ws = torch.empty(lib.wnb_resblock_bwd_workspace(B, T, R, S, Ap, ks) // 4, device="cuda")
    dx = torch.empty(B, T, R, device="cuda")
    dh = torch.zeros(B, T, Ap, device="cuda")
    dw1, db1 = torch.zeros(2 * R, K1, device="cuda"), torch.zeros(2 * R, device="cuda")
    dw2, db2 = torch.zeros(R + S, R, device="cuda"), torch.zeros(R + S, device="cuda")
    _lib.check(lib.wnb_resblock_bwd(_lib.ptr(xin), _lib.ptr(haux), _lib.ptr(dout), _lib.ptr(dskip), _lib.ptr(W1),
                                    _lib.ptr(b1), _lib.ptr(w1t), _lib.ptr(w2t), _lib.ptr(dx), _lib.ptr(dh),
                                    _lib.ptr(dw1), _lib.ptr(db1), _lib.ptr(dw2), _lib.ptr(db2), _lib.ptr(ws),
                                    B, T, R, S, Ap, ks, d, mode, _lib.stream()), "resblock_bwd")
    torch.cuda.synchronize()
    return dict(xout=xout, skip=skip, dx=dx, dh=dh, dw1=dw1, db1=db1, dw2=dw2, db2=db2)


@pytest.mark.parametrize("R,S,Ap,ks,d,T,last,init", [
    (128, 256, 32, 2, 4, 300, False, True),      # mixed [dout | dskip] wgrad block is not needed (R % 128 == 0)
    (512, 256, 32, 2, 16, 520, False, False),    # the recipes' shape (egs/arctic/sd/run.sh:48-49)
    (128, 64, 96, 3, 2, 260, False, False),      # kernel_size 3, 80-dim aux padded to 96 (ljspeech-like)
    (192, 512, 32, 2, 1, 256, True, False),      # R % 128 != 0: mixed wgrad block, last layer (no dout)
    (192, 96, 32, 3, 8, 200, False, True),
])
def test_composed_block_fwd_bwd_tf32_vs_fp32(R, S, Ap, ks, d, T, last, init):
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    assert lib.wnb_resblock_fwd_supported(R, S, Ap, ks, _lib.MATH_TF32) == 2
    ref = _block_general(_lib.MATH_FP32, R, S, Ap, ks, d, 2, T, last, init, seed=R + S + T)
    got = _block_general(_lib.MATH_TF32, R, S, Ap, ks, d, 2, T, last, init, seed=R + S + T)
    for k, r in ref.items():
        if r is None:
            continue
        g = got[k]
        assert torch.isfinite(g).all(), k
        rel = (g - r).norm().item() / max(r.norm().item(), 1e-12)
        assert rel < 6e-3, (k, rel)


def test_composed_full_model_step_tf32_vs_fp32():
    """ljspeech-like small model (80-dim aux, kernel_size 3, R=128/S=64): tf32 (composed tensor-core path) vs fp32."""
    from pytorchwavenetvocoder_b200.nets import cross_entropy
    from pytorchwavenetvocoder_b200.nets.wavenet import tc_supported
    cfg_t = (256, 80, 128, 64, 4, 2, 3, 8)
    assert tc_supported(cfg_t)
    cfg = O.Config(*cfg_t)
    p = O.make_params(cfg, 9)
    rng = np.random.RandomState(3)
    B, T = 2, 384
    x = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    t = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    h = torch.from_numpy(rng.standard_normal((B, 80, T // 8)).astype(np.float32)).cuda()
    res = {}
    for mode in ("fp32", "tf32"):
        net = our_model(cfg, p, math_mode=mode).train()
        y = net(x, h)
        loss = cross_entropy(y, t, cfg.receptive_field)
        loss.backward()
        res[mode] = (loss.item(), y.detach(), {k: v.grad.clone() for k, v in net.named_parameters() if v.grad is not None})
    assert abs(res["fp32"][0] - res["tf32"][0]) < 2e-3
    assert (res["fp32"][1] - res["tf32"][1]).abs().max().item() < 5e-2
    for k, g in res["fp32"][2].items():
        g2 = res["tf32"][2][k]
        if g.numel() == 1:
            assert (g - g2).abs().item() <= 3e-3, k
        else:
            tol = 0.10 if g.dim() == 1 else 0.08     # K = 3*128+96 per gate GEMM: a little more tf32 rounding
            assert (g - g2).norm().item() <= tol * g.norm().item() + 1e-7, k


# ------------------------------------------------------------------------------------------
# deferred-skip stack (csrc/stack.cu, resblock_z.cu) against the per-block formulation
# (the block kernel and the skip GEMM alone are checked element-wise in test_gpu_tc_stages.py)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,depth,repeat,B,T", [
    (512, 5, 2, 3, 1040),     # T not a multiple of the 128-row tile; CTAs of the segmented dW launches span two blocks
    (256, 7, 1, 2, 700),      # L*R = 448: dZ_all in 64-column blocks, dWskip in 7 column groups
    (96, 3, 1, 1, 333),       # S not a multiple of 128: zero-filled rows in the dWskip M-block
    (512, 3, 2, 1, 100),      # 2 time tiles per block: every CTA of the segmented dW1 / dW2res launch walks through
                              # all six blocks and recycles both accumulator sets
])
def test_deferred_skip_stack_matches_per_block_training_step(S, depth, repeat, B, T):
    """Same model, same batch: WaveNet.forward/backward through the deferred-skip stack (one ABI call per
    direction) vs the per-block tf32 path.  Both are tf32; they differ only in summation order, so logits agree to
    2e-3 abs and every gradient to 3 % (relative Frobenius norm; bias gradients 5 %) -- the gradients at the bottom
    of the stack carry the tf32 rounding of every block above them in both runs."""
    from pytorchwavenetvocoder_b200.nets import cross_entropy
    cfg = O.Config(256, 28, 64, S, depth, repeat, 2, 0)
    p = O.make_params(cfg, 21)
    rng = np.random.RandomState(4)
    x = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    t = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    h = torch.from_numpy(rng.standard_normal((B, 28, T)).astype(np.float32)).cuda()
    res = {}
    for deferred in (False, True):
        net = our_model(cfg, p, math_mode="tf32").train()
        net.deferred_skip = deferred
        y = net(x, h)
        loss = cross_entropy(y, t, min(32, T // 4))
        loss.backward()
        res[deferred] = (y.detach().clone(), loss.item(),
                         {k: (None if v.grad is None else v.grad.clone()) for k, v in net.named_parameters()})
    assert (res[True][0] - res[False][0]).abs().max().item() <= 2e-3
    assert abs(res[True][1] - res[False][1]) < 2e-4
    for k, g in res[False][2].items():
        g2 = res[True][2][k]
        assert (g is None) == (g2 is None), k          # the last block's res_1x1 has no gradient in either form
        if g is None:
            continue
        if g.numel() == 1:
            assert (g - g2).abs().item() <= 3e-3, k
        else:
            tol = 0.05 if g.dim() == 1 else 0.03
            assert (g - g2).norm().item() <= tol * g.norm().item() + 1e-7, (k, (g - g2).norm().item(), g.norm().item())


def test_deferred_skip_inference_ping_pong():
    """No-grad forward uses two residual buffers (nxs = 2) instead of L: same logits as the training-mode forward."""
    cfg = O.Config(256, 28, 64, 256, 4, 2, 2, 0)
    p = O.make_params(cfg, 2)
    rng = np.random.RandomState(9)
    B, T = 2, 700
    x = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    h = torch.from_numpy(rng.standard_normal((B, 28, T)).astype(np.float32)).cuda()
    net = our_model(cfg, p, math_mode="tf32")
    with torch.no_grad():
        y0 = net(x, h)
    y1 = net.train()(x, h)
    assert torch.equal(y0, y1.detach())
