# -*- coding: utf-8 -*-
"""H100-native mirror of ``wavenet_vocoder/nets/wavenet.py`` (reference v0.1.1).

Same import surface, constructor arguments, attributes, method signatures, ``state_dict`` keys and
error behaviour as the reference module (SURVEY.md 8b), but every hot-path computation is a
hand-written sm_90a kernel reached through the C ABI in ``include/wnb200.h``:

* ``WaveNet.forward``  (reference wavenet.py:212-241)  -> front gather, aux up-sampling, ONE fused
  kernel per residual block, post network; backward through ``torch.autograd.Function``.
* ``fast_generate`` / ``batch_fast_generate`` (wavenet.py:309-511) -> one persistent kernel launch, run as a
  ``DecodeSession`` given every aux frame in one call (the same object decodes chunk by chunk as frames arrive).
* ``encode_mu_law`` / ``decode_mu_law`` (wavenet.py:17-47) -> device kernels, numpy in / numpy out.

PyTorch only owns the memory, the parameters and the streams.  There is no CPU fallback: calling the
model with CPU tensors raises.
"""
import collections
import ctypes
import logging
import math
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib
from .._lib import MATH_BF16, MATH_FP32, MATH_TF32, MODE_ARGMAX, MODE_SAMPLING, check, ptr, stream

__all__ = ["encode_mu_law", "decode_mu_law", "initialize", "OneHot", "CausalConv1d", "UpSampling",
           "WaveNet", "cross_entropy", "mulaw_pcm16_table", "codes_to_pcm16", "DecodeSession", "DecodePool",
           "decode_window"]

# bench.py sets this to a list to get (start, end) CUDA-event pairs around every fused-block launch
PROFILE_EVENTS = None


def tc_supported(cfg):
    """True when the tf32 tensor-core path covers WaveNet(*cfg)."""
    lib = _lib.load()
    Q, A, R, S, depth, repeat, ks, U = cfg
    return bool(lib.wnb_resblock_fwd_supported(R, S, _round_up(A, 32), ks, MATH_TF32))


def bf16_supported(cfg):
    """True when the bf16 tensor-core path (math_mode="bf16": the composed per-block GEMMs and the post network)
    covers WaveNet(*cfg)."""
    lib = _lib.load()
    Q, A, R, S, depth, repeat, ks, U = cfg
    ok = S % 32 == 0 and Q % 32 == 0 and (S <= 256 or S == 512) and (Q <= 256 or Q == 512)
    return ok and lib.wnb_resblock_fwd_supported(R, S, _round_up(A, 32), ks, MATH_BF16) == 2


def decode_bf16_supported(cfg):
    """True when the opt-in bf16 tensor-core decoder (decode_math="bf16", csrc/decode_bf16.cu) covers WaveNet(*cfg)."""
    lib = _lib.load()
    Q, A, R, S, depth, repeat, ks, U = cfg
    return bool(lib.wnb_decode_bf16_supported(Q, _round_up(A, 32), R, S, ks, depth * repeat))


def _bf16_swizzle(t):
    """(..., N, K) -> (..., K/64, N, 64): K split into 64-wide tiles, each tile in the 128B swizzle of the wgmma B operand
    (element (n, k) at column ((k // 8) ^ (n % 8)) * 8 + k % 8 of row n)."""
    *lead, N, K = t.shape
    t = t.reshape(*lead, N, K // 64, 64).transpose(-3, -2)
    k = torch.arange(64, device=t.device)
    n = torch.arange(N, device=t.device)[:, None]
    dst = (((k >> 3) ^ (n & 7)) << 3) + (k & 7)
    out = torch.empty_like(t)
    out.scatter_(-1, dst.expand_as(t), t)
    return out


def _device():
    if not torch.cuda.is_available():
        raise _lib.WnbError("no CUDA device: the wnb200 kernels need a CUDA GPU (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


# ------------------------------------------------------------------------------------------
# mu-law (reference wavenet.py:17-47): numpy in, numpy out, computed on the GPU
# ------------------------------------------------------------------------------------------
def encode_mu_law(x, mu=256):
    """PERFORM MU-LAW ENCODING (reference wavenet.py:17-30).

    Args:
        x (ndarray): Audio signal with the range from -1 to 1 (float32 or float64).
        mu (int): Quantized level.

    Returns:
        ndarray: int64 quantized signal with the range from 0 to mu - 1.
    """
    lib = _lib.load()
    x = np.asarray(x)
    if x.dtype not in (np.float32, np.float64):
        x = x.astype(np.float64)
    dev = _device()
    xt = torch.from_numpy(np.ascontiguousarray(x).reshape(-1)).to(dev)
    yt = torch.empty(xt.numel(), dtype=torch.int64, device=dev)
    fn = lib.wnb_mulaw_encode_f32 if x.dtype == np.float32 else lib.wnb_mulaw_encode_f64
    check(fn(ptr(xt), ptr(yt), xt.numel(), int(mu), stream()), "mulaw_encode")
    return yt.cpu().numpy().reshape(x.shape)


def decode_mu_law(y, mu=256):
    """PERFORM MU-LAW DECODING (reference wavenet.py:33-47); returns float64 like numpy does."""
    lib = _lib.load()
    y = np.asarray(y)
    dev = _device()
    yt = torch.from_numpy(np.ascontiguousarray(y).astype(np.int64).reshape(-1)).to(dev)
    xt = torch.empty(yt.numel(), dtype=torch.float64, device=dev)
    check(lib.wnb_mulaw_decode_f64(ptr(yt), ptr(xt), yt.numel(), int(mu), stream()), "mulaw_decode")
    return xt.cpu().numpy().reshape(y.shape)


def mulaw_pcm16_table(mu=256):
    """int16 PCM value of every mu-law code: ``decode_mu_law`` (reference wavenet.py:33-47) followed by the PCM_16
    quantisation of ``utils.write_wav``'s stdlib writer (round-half-even of x * 32768, clipped to int16)."""
    x = decode_mu_law(np.arange(mu), mu)
    return np.clip(np.round(x * 32768.0), -32768, 32767).astype(np.int16)


def codes_to_pcm16(codes, mu=256):
    """(B, n) int32 CUDA tensor of generated codes -> (B, n) int16 CUDA tensor (one gather kernel for the whole batch)."""
    lib = _lib.load()
    codes = codes.contiguous()
    if codes.dtype != torch.int32:
        codes = codes.to(torch.int32)
    tab = torch.from_numpy(mulaw_pcm16_table(mu)).to(codes.device)
    out = torch.empty(codes.shape, dtype=torch.int16, device=codes.device)
    check(lib.wnb_lut_i16(ptr(codes), ptr(tab), ptr(out), codes.numel(), int(mu), stream()), "lut_i16")
    return out


def initialize(m):
    """INITILIZE CONV WITH XAVIER (reference wavenet.py:50-63)."""
    if isinstance(m, nn.Conv1d):
        nn.init.xavier_uniform_(m.weight)
        nn.init.constant_(m.bias, 0.0)
    if isinstance(m, nn.ConvTranspose2d):
        nn.init.constant_(m.weight, 1.0)
        nn.init.constant_(m.bias, 0.0)


# ------------------------------------------------------------------------------------------
# autograd functions wrapping the C ABI
# ------------------------------------------------------------------------------------------
class _UpsampleFn(torch.autograd.Function):
    """aux up-sampling + (B,A,Tf)->(B,T,Ap) layout change (reference wavenet.py:124-154)."""

    @staticmethod
    def forward(ctx, h, w, b, Ap):
        lib = _lib.load()
        h = h.contiguous().float()
        B, A, Tf = h.shape
        U = 0 if w is None else w.numel()
        T = Tf * U if U > 0 else Tf
        out = torch.empty(B, T, Ap, device=h.device, dtype=torch.float32)
        wc = None if w is None else w.contiguous().view(-1)
        bc = None if b is None else b.contiguous().view(-1)
        check(lib.wnb_aux_upsample_fwd(ptr(h), ptr(wc), ptr(bc), ptr(out), B, A, Ap, Tf, U, stream()),
              "aux_upsample_fwd")
        ctx.save_for_backward(h)
        ctx.meta = (B, A, Ap, Tf, U, None if w is None else w.shape, None if b is None else b.shape)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = _lib.load()
        (h,) = ctx.saved_tensors
        B, A, Ap, Tf, U, wshape, bshape = ctx.meta
        if U == 0:
            return None, None, None, None
        dout = dout.contiguous()
        dw = torch.zeros(U, device=h.device, dtype=torch.float32)
        db = torch.zeros(1, device=h.device, dtype=torch.float32)
        check(lib.wnb_aux_upsample_bwd(ptr(h), ptr(dout), ptr(dw), ptr(db), B, A, Ap, Tf, U, stream()),
              "aux_upsample_bwd")
        return None, dw.view(wshape), db.view(bshape), None


class _CrossEntropyFn(torch.autograd.Function):
    """CrossEntropyLoss(mean) over logits[:, start:] fused with its gradient (bin/train.py:534-536)."""

    @staticmethod
    def forward(ctx, logits, target, start):
        lib = _lib.load()
        logits = logits.contiguous()
        target = target.contiguous()
        B, T, Q = logits.shape
        if target.dtype != torch.int64 or tuple(target.shape) != (B, T) or target.device != logits.device:
            raise ValueError("cross_entropy: target should be an int64 (B, T) = %s tensor on %s, got %s %s on %s"
                             % ((B, T), logits.device, target.dtype, tuple(target.shape), target.device))
        loss = torch.zeros(1, device=logits.device, dtype=torch.float64)
        need = ctx.needs_input_grad[0]
        dl = torch.empty_like(logits) if need else None
        check(lib.wnb_cross_entropy(ptr(logits), ptr(target), ptr(loss), ptr(dl), B, T, Q, int(start), stream()),
              "cross_entropy")
        ctx.dl = dl
        return loss[0].float()

    @staticmethod
    def backward(ctx, g):
        dl = ctx.dl
        ctx.dl = None
        return dl * g, None, None


def cross_entropy(logits, target, start=0):
    """Mean cross entropy over ``logits[:, start:]`` (B,T,Q) vs ``target[:, start:]`` (B,T)."""
    return _CrossEntropyFn.apply(logits, target, start)


class _WaveNetFn(torch.autograd.Function):
    """WaveNet.forward (reference wavenet.py:212-241) on packed weights."""

    @staticmethod
    def forward(ctx, x, haux, wf, bf, W1, b1, W2, b2, Wp1, bp1, Wp2, bp2, meta):
        lib = _lib.load()
        Q, R, S, Ap, ks, dilations, math_mode = meta
        B, T = x.shape
        L = len(dilations)
        dev = x.device
        x = x.contiguous()
        need_grad = any(ctx.needs_input_grad)
        st = stream()
        # residual-stream buffers: all L layer inputs are kept when a backward will follow
        # (the gate is recomputed there, nothing else is saved per layer); otherwise ping-pong.
        nbuf = L if need_grad else min(L, 2)
        xs = torch.empty(nbuf, B, T, R, device=dev, dtype=torch.float32)
        check(lib.wnb_front_embed_fwd(ptr(x), ptr(wf), ptr(bf), ptr(xs[0]), B, T, Q, R, ks, st), "front_embed_fwd")
        skip = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        # the composed tensor-core path (tf32 or bf16) needs a z scratch
        zbuf = None
        if math_mode in (MATH_TF32, MATH_BF16) and lib.wnb_resblock_fwd_supported(R, S, Ap, ks, math_mode) == 2:
            zbuf = torch.empty(B, T, R, device=dev, dtype=torch.float32)
        prof = PROFILE_EVENTS
        for l, d in enumerate(dilations):
            xin = xs[l % nbuf]
            xout = xs[(l + 1) % nbuf] if l + 1 < L else None
            if prof is not None:
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                ev[0].record()
            check(lib.wnb_resblock_fwd(ptr(xin), ptr(haux), ptr(W1[l]), ptr(b1[l]), ptr(W2[l]), ptr(b2[l]),
                                       ptr(xout), ptr(skip), ptr(zbuf), B, T, R, S, Ap, ks, int(d),
                                       1 if l == 0 else 0, math_mode, st), "resblock_fwd")
            if prof is not None:
                ev[1].record()
                prof.append(ev)
        r1 = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        logits = torch.empty(B, T, Q, device=dev, dtype=torch.float32)
        check(lib.wnb_post_fwd(ptr(skip), ptr(Wp1), ptr(bp1), ptr(Wp2), ptr(bp2), ptr(r1), ptr(logits),
                               B, T, S, Q, math_mode, 0, st), "post_fwd")
        if need_grad:
            ctx.save_for_backward(x, haux, wf, W1, b1, W2, Wp1, Wp2, xs, skip, r1)
            ctx.meta = meta
            ctx.haux_needs_grad = ctx.needs_input_grad[1]
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        lib = _lib.load()
        x, haux, wf, W1, b1, W2, Wp1, Wp2, xs, skip, r1 = ctx.saved_tensors
        Q, R, S, Ap, ks, dilations, math_mode = ctx.meta
        B, T = x.shape
        L = len(dilations)
        dev = x.device
        st = stream()
        dlogits = dlogits.contiguous()
        z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float32)  # noqa: E731
        K1 = ks * R + Ap
        dWp1, dbp1, dWp2, dbp2 = z(S, S), z(S), z(Q, S), z(Q)
        dskip = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        ws_post = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        wp1t = Wp1.t().contiguous()
        wp2t = Wp2.t().contiguous()
        check(lib.wnb_post_bwd(ptr(skip), ptr(r1), ptr(dlogits), ptr(wp1t), ptr(wp2t), ptr(dskip), ptr(dWp1),
                               ptr(dbp1), ptr(dWp2), ptr(dbp2), ptr(ws_post), B, T, S, Q, math_mode, st), "post_bwd")
        del ws_post
        dW1, db1, dW2, db2 = z(L, 2 * R, K1), z(L, 2 * R), z(L, R + S, R), z(L, R + S)
        dhaux = z(B, T, Ap) if ctx.haux_needs_grad else None
        w1t = W1.transpose(1, 2).contiguous()   # (L, K1, 2R)
        w2t = W2.transpose(1, 2).contiguous()   # (L, R, R+S)
        nbytes = lib.wnb_resblock_bwd_workspace(B, T, R, S, Ap, ks)
        ws = torch.empty(nbytes // 4, device=dev, dtype=torch.float32)
        dbuf = [torch.empty(B, T, R, device=dev, dtype=torch.float32) for _ in range(2)]
        dout = None
        for l in reversed(range(L)):
            dxin = dbuf[l % 2]
            check(lib.wnb_resblock_bwd(ptr(xs[l]), ptr(haux), ptr(dout), ptr(dskip), ptr(W1[l]), ptr(b1[l]),
                                       ptr(w1t[l]), ptr(w2t[l]), ptr(dxin), ptr(dhaux), ptr(dW1[l]), ptr(db1[l]),
                                       ptr(dW2[l]), ptr(db2[l]), ptr(ws), B, T, R, S, Ap, ks, int(dilations[l]),
                                       math_mode, st), "resblock_bwd")
            dout = dxin
        dwf, dbf = z(ks, Q, R), z(R)
        check(lib.wnb_front_embed_bwd(ptr(x), ptr(dout), ptr(dwf), ptr(dbf), B, T, Q, R, ks, st), "front_embed_bwd")
        return None, dhaux, dwf, dbf, dW1, db1, dW2, db2, dWp1, dbp1, dWp2, dbp2, None


class _WaveNetStackFn(torch.autograd.Function):
    """WaveNet.forward (reference wavenet.py:212-241) with the skip path in deferred form (csrc/stack.cu): the blocks
    write their gate outputs z_l into Z_all (B,T,L*R) and ONE GEMM forms skip = Z_all Wskip^T + bskip; the backward
    hoists dZ_all = dskip Wskip and dWskip = dskip^T Z_all out of the block loop the same way.  Same numbers as the
    per-block form (different summation order inside tf32/fp32 accumulation only)."""

    @staticmethod
    def forward(ctx, x, haux, wf, bf, W1, b1, W2res, b2res, Wskip, bskip, Wp1, bp1, Wp2, bp2, meta):
        lib = _lib.load()
        Q, R, S, Ap, ks, dilations, math_mode = meta
        B, T = x.shape
        L = len(dilations)
        dev = x.device
        x = x.contiguous()
        need_grad = any(ctx.needs_input_grad)
        st = stream()
        nbuf = L if need_grad else min(L, 2)
        xs = torch.empty(nbuf, B, T, R, device=dev, dtype=torch.float32)
        check(lib.wnb_front_embed_fwd(ptr(x), ptr(wf), ptr(bf), ptr(xs[0]), B, T, Q, R, ks, st), "front_embed_fwd")
        zall = torch.empty(B, T, L * R, device=dev, dtype=torch.float32)
        skip = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        dil = (ctypes.c_int * L)(*[int(d) for d in dilations])
        prof = PROFILE_EVENTS
        if prof is None:
            check(lib.wnb_stack_fwd(ptr(xs), nbuf, ptr(haux), ptr(W1), ptr(b1), ptr(W2res), ptr(b2res), ptr(Wskip),
                                    ptr(bskip), ptr(zall), ptr(skip), dil, L, B, T, R, S, Ap, ks, 1, st), "stack_fwd")
        else:   # same launches, one ABI call per block so that each can be bracketed by CUDA events
            for l, d in enumerate(dilations):
                xout = xs[(l + 1) % nbuf] if l + 1 < L else None
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                ev[0].record()
                check(lib.wnb_resblock_fwd_z(ptr(xs[l % nbuf]), ptr(haux), ptr(W1[l]), ptr(b1[l]), ptr(W2res[l]),
                                             ptr(b2res[l]), ptr(xout), ptr(zall), L * R, l * R, B, T, R, Ap, ks,
                                             int(d), st), "resblock_fwd_z")
                ev[1].record()
                prof.append(ev)
            check(lib.wnb_skip_gemm(ptr(zall), ptr(Wskip), ptr(bskip), ptr(skip), B, T, L * R, S, 1, st), "skip_gemm")
        r1 = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        logits = torch.empty(B, T, Q, device=dev, dtype=torch.float32)
        check(lib.wnb_post_fwd(ptr(skip), ptr(Wp1), ptr(bp1), ptr(Wp2), ptr(bp2), ptr(r1), ptr(logits),
                               B, T, S, Q, math_mode, 1, st), "post_fwd")
        if need_grad:
            ctx.save_for_backward(x, haux, wf, W1, b1, W2res, Wskip, Wp1, Wp2, xs, zall, skip, r1)
            ctx.meta = meta
            ctx.haux_needs_grad = ctx.needs_input_grad[1]
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        lib = _lib.load()
        x, haux, wf, W1, b1, W2res, Wskip, Wp1, Wp2, xs, zall, skip, r1 = ctx.saved_tensors
        Q, R, S, Ap, ks, dilations, math_mode = ctx.meta
        B, T = x.shape
        L = len(dilations)
        dev = x.device
        st = stream()
        dlogits = dlogits.contiguous()
        z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float32)  # noqa: E731
        K1 = ks * R + Ap
        dWp1, dbp1, dWp2, dbp2 = z(S, S), z(S), z(Q, S), z(Q)
        dskip = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        ws_post = torch.empty(B, T, S, device=dev, dtype=torch.float32)
        wp1t = Wp1.t().contiguous()
        wp2t = Wp2.t().contiguous()
        check(lib.wnb_post_bwd(ptr(skip), ptr(r1), ptr(dlogits), ptr(wp1t), ptr(wp2t), ptr(dskip), ptr(dWp1),
                               ptr(dbp1), ptr(dWp2), ptr(dbp2), ptr(ws_post), B, T, S, Q, math_mode, st), "post_bwd")
        del ws_post
        dW1, db1, dW2res, db2res = z(L, 2 * R, K1), z(L, 2 * R), z(L, R, R), z(L, R)
        dWskip, dbskip = z(S, L * R), z(S)
        dhaux = z(B, T, Ap) if ctx.haux_needs_grad else None
        w1t = W1.transpose(1, 2).contiguous()         # (L, K1, 2R)
        wgate = torch.zeros(L, 3 * R, K1 + R, device=dev, dtype=torch.float32)   # [[W1, 0], [0, W2res^T]]
        wgate[:, :2 * R, :K1] = W1
        wgate[:, 2 * R:, K1:] = W2res.transpose(1, 2)
        wskt = Wskip.t().contiguous()                 # (L*R, S)
        nbytes = lib.wnb_stack_bwd_workspace(L, B, T, R, S, Ap, ks)
        ws = torch.empty(nbytes // 4, device=dev, dtype=torch.float32)
        dx0 = torch.empty(B, T, R, device=dev, dtype=torch.float32)
        dil = (ctypes.c_int * L)(*[int(d) for d in dilations])
        check(lib.wnb_stack_bwd(ptr(xs), ptr(haux), ptr(zall), ptr(dskip), ptr(W1), ptr(b1), ptr(w1t), ptr(wgate),
                                ptr(wskt), ptr(dx0), ptr(dhaux), ptr(dW1), ptr(db1), ptr(dW2res), ptr(db2res),
                                ptr(dWskip), ptr(dbskip), ptr(ws), dil, L, B, T, R, S, Ap, ks, st), "stack_bwd")
        del ws
        dwf, dbf = z(ks, Q, R), z(R)
        check(lib.wnb_front_embed_bwd(ptr(x), ptr(dx0), ptr(dwf), ptr(dbf), B, T, Q, R, ks, st), "front_embed_bwd")
        return (None, dhaux, dwf, dbf, dW1, db1, dW2res, db2res, dWskip, dbskip, dWp1, dbp1, dWp2, dbp2, None)


class _StackTrainFn(torch.autograd.Function):
    """WaveNet.forward (reference wavenet.py:212-241) [+ the cross entropy of bin/train.py:534-536] on the deferred-skip
    stack, with NO torch arithmetic in between: parameters are packed by ``wnb_pack_weights`` (one launch), the packed
    gradients are scattered into one flat buffer by the same kernel (one launch) and handed to autograd as views, so
    ``p.grad`` of every parameter aliases one contiguous tensor (``module._wnb_flat_grad``: what the data-parallel
    all-reduce sends).  ``target is None``: returns the (B,T,Q) logits; otherwise the mean CE over ``[:, start:]``."""

    @staticmethod
    def forward(ctx, net, plan, x, h, target, start, *params):
        lib = _lib.load()
        d = plan.dims
        R, S, Q, ks, A, Ap, L, U = d["R"], d["S"], d["Q"], d["ks"], d["A"], d["Ap"], d["L"], d["U"]
        dev = x.device
        st = stream()
        x = x.contiguous()
        h = h.contiguous().float()
        B, T = x.shape
        Tf = h.size(2)
        if h.size(1) != A:
            raise ValueError("aux feature has %d dims, expected %d" % (h.size(1), A))
        if (Tf * U if U > 0 else Tf) != T:
            raise ValueError("aux length %d does not match waveform length %d" % (Tf * max(U, 1), T))
        need_grad = any(ctx.needs_input_grad)
        plan.pack(st)
        P = plan.p
        f32 = dict(device=dev, dtype=torch.float32)
        haux = torch.empty(B, T, Ap, **f32)
        upw = net.upsampling.conv.weight if U > 0 else None
        upb = net.upsampling.conv.bias if U > 0 else None
        check(lib.wnb_aux_upsample_fwd(ptr(h), ptr(upw), ptr(upb), ptr(haux), B, A, Ap, Tf, U, st), "aux_upsample_fwd")
        nbuf = L if need_grad else min(L, 2)
        xs = torch.empty(nbuf, B, T, R, **f32)
        check(lib.wnb_front_embed_fwd(ptr(x), ptr(P("wf")), ptr(P("bf")), ptr(xs[0]), B, T, Q, R, ks, st), "front_embed_fwd")
        zall = torch.empty(B, T, L * R, **f32)
        skip = torch.empty(B, T, S, **f32)
        dil = (ctypes.c_int * L)(*[int(v) for v in net.dilations])
        check(lib.wnb_stack_fwd(ptr(xs), nbuf, ptr(haux), ptr(P("W1")), ptr(P("b1")), ptr(P("W2res")), ptr(P("b2res")),
                                ptr(P("Wskip")), ptr(P("bskip")), ptr(zall), ptr(skip), dil, L, B, T, R, S, Ap, ks, 1, st),
              "stack_fwd")
        r1 = torch.empty(B, T, S, **f32)
        logits = torch.empty(B, T, Q, **f32)
        check(lib.wnb_post_fwd(ptr(skip), ptr(P("Wp1")), ptr(P("bp1")), ptr(P("Wp2")), ptr(P("bp2")), ptr(r1), ptr(logits),
                               B, T, S, Q, MATH_TF32, 1, st), "post_fwd")
        dbg = getattr(net, "_wnb_debug", None)
        if dbg is not None:     # test aid: the ReLU sign patterns of the post network (tests/test_gpu_oracle_direct.py)
            dbg["skip_mask"], dbg["r1_mask"] = skip > 0, r1 > 0
        out = logits
        dl = None
        if target is not None:
            target = target.contiguous()
            if target.dtype != torch.int64 or tuple(target.shape) != (B, T) or target.device != dev:
                raise ValueError("target should be an int64 (B, T) tensor on the model's device")
            loss = torch.empty(1, device=dev, dtype=torch.float64)
            check(lib.wnb_zero(ptr(loss), 8, st), "zero")
            dl = logits if need_grad else None     # dlogits overwrite the logits in place (each row is read, then written)
            check(lib.wnb_cross_entropy(ptr(logits), ptr(target), ptr(loss), ptr(dl), B, T, Q, int(start), st),
                  "cross_entropy")
            out = loss.float().view(())
        if need_grad:
            ctx.save_for_backward(x, h, haux, xs, zall, skip, r1)
            ctx.net, ctx.plan, ctx.dl, ctx.dil = net, plan, dl, dil
            ctx.fused_loss = target is not None
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        x, h, haux, xs, zall, skip, r1 = ctx.saved_tensors
        net, plan, dil = ctx.net, ctx.plan, ctx.dil
        d = plan.dims
        R, S, Q, ks, A, Ap, L, U = d["R"], d["S"], d["Q"], d["ks"], d["A"], d["Ap"], d["L"], d["U"]
        B, T = x.shape
        Tf = h.size(2)
        dev = x.device
        st = stream()
        f32 = dict(device=dev, dtype=torch.float32)
        if ctx.fused_loss:
            dlogits, scale = ctx.dl, g.contiguous().float()   # d loss / d logits from the CE kernel; g scales the result
            ctx.dl = None
        else:
            dlogits, scale = g.contiguous(), None
        P = plan.p
        gbuf = torch.empty(plan.G.size, **f32)
        check(lib.wnb_zero(ptr(gbuf), gbuf.numel() * 4, st), "zero")
        G = lambda name: plan.G.view(gbuf, name)  # noqa: E731
        dskip = torch.empty(B, T, S, **f32)
        ws_post = torch.empty(B, T, S, **f32)
        check(lib.wnb_post_bwd(ptr(skip), ptr(r1), ptr(dlogits), ptr(P("wp1t")), ptr(P("wp2t")), ptr(dskip), ptr(G("Wp1")),
                               ptr(G("bp1")), ptr(G("Wp2")), ptr(G("bp2")), ptr(ws_post), B, T, S, Q, MATH_TF32, st),
              "post_bwd")
        del ws_post, dlogits
        dhaux = None
        if U > 0:
            dhaux = torch.empty(B, T, Ap, **f32)
            check(lib.wnb_zero(ptr(dhaux), dhaux.numel() * 4, st), "zero")
        nbytes = lib.wnb_stack_bwd_workspace(L, B, T, R, S, Ap, ks)
        ws = torch.empty(nbytes // 4, **f32)
        dx0 = torch.empty(B, T, R, **f32)
        check(lib.wnb_stack_bwd(ptr(xs), ptr(haux), ptr(zall), ptr(dskip), ptr(P("W1")), ptr(P("b1")), ptr(P("w1t")),
                                ptr(P("wgate")), ptr(P("wskt")), ptr(dx0), ptr(dhaux), ptr(G("W1")), ptr(G("b1")),
                                ptr(G("W2res")), ptr(G("b2res")), ptr(G("Wskip")), ptr(G("bskip")), ptr(ws), dil, L, B, T,
                                R, S, Ap, ks, st), "stack_bwd")
        del ws
        check(lib.wnb_front_embed_bwd(ptr(x), ptr(dx0), ptr(G("wf")), ptr(G("bf")), B, T, Q, R, ks, st), "front_embed_bwd")
        if U > 0:
            check(lib.wnb_aux_upsample_bwd(ptr(h), ptr(dhaux), ptr(G("upw")), ptr(G("upb")), B, A, Ap, Tf, U, st),
                  "aux_upsample_bwd")
        flat = torch.empty(plan.grad_size, **f32)
        plan.unpack(gbuf, flat, scale, st)
        net._wnb_flat_grad = flat
        return (None, None, None, None, None, None) + tuple(plan.grad_views(flat))


# ------------------------------------------------------------------------------------------
# modules (same names / parameters / state_dict keys as the reference)
# ------------------------------------------------------------------------------------------
class OneHot(nn.Module):
    """CONVERT TO ONE-HOT VECTOR (reference wavenet.py:66-92).

    Kept for API compatibility only: ``WaveNet`` never materialises the one-hot tensor (the front
    convolution is an embedding gather on the device)."""

    def __init__(self, depth):
        super(OneHot, self).__init__()
        self.depth = depth

    def forward(self, x):
        x = x % self.depth
        x = torch.unsqueeze(x, 2)
        x_onehot = x.new_zeros(x.size(0), x.size(1), self.depth).float()
        return x_onehot.scatter_(2, x, 1)


class CausalConv1d(nn.Module):
    """1D DILATED CAUSAL CONVOLUTION (reference wavenet.py:95-121): parameter container.

    Inside ``WaveNet`` these weights are consumed by the fused block kernel; the module keeps the
    reference's ``.conv.weight`` / ``.conv.bias`` parameter names so checkpoints interchange."""

    def __init__(self, in_channels, out_channels, kernel_size, dilation=1, bias=True):
        super(CausalConv1d, self).__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = kernel_size
        self.dilation = dilation
        self.padding = padding = (kernel_size - 1) * dilation
        self.conv = nn.Conv1d(in_channels, out_channels, kernel_size,
                              padding=padding, dilation=dilation, bias=bias)

    def forward(self, x):
        """FORWARD CALCULATION (reference wavenet.py:108-121): x (B, C, T) -> (B, C_out, T), inference only.

        Inside ``WaveNet`` the convolution runs in the fused block kernels; this standalone form exists for API
        compatibility and goes through ``wnb_causal_conv1d_fwd`` (no autograd)."""
        if torch.is_grad_enabled() and (x.requires_grad or self.conv.weight.requires_grad):
            # the reference module is a differentiable Conv1d; this standalone helper has no backward kernel, and a
            # silently detached result would train nothing -- say so instead
            raise RuntimeError("CausalConv1d.forward is inference-only in this build (no standalone backward): "
                               "call it under torch.no_grad(); training goes through WaveNet.forward")
        lib = _lib.load()
        if not x.is_cuda:
            raise _lib.WnbError("CausalConv1d.forward needs CUDA tensors: this build has no CPU fallback")
        B, C, T = x.shape
        xl = x.detach().float().transpose(1, 2).contiguous()                                   # (B, T, C)
        w = self.conv.weight.detach().float().permute(0, 2, 1).reshape(self.out_channels, -1).contiguous()  # [o][j*C+c]
        b = None if self.conv.bias is None else self.conv.bias.detach().float().contiguous()
        out = torch.empty(B, T, self.out_channels, device=x.device, dtype=torch.float32)
        check(lib.wnb_causal_conv1d_fwd(ptr(xl), ptr(w), ptr(b), ptr(out), B, T, C, self.out_channels,
                                        self.kernel_size, self.dilation, stream()), "causal_conv1d_fwd")
        return out.transpose(1, 2)


class UpSampling(nn.Module):
    """UPSAMPLING LAYER WITH DECONVOLUTION (reference wavenet.py:124-154)."""

    def __init__(self, upsampling_factor, bias=True):
        super(UpSampling, self).__init__()
        self.upsampling_factor = upsampling_factor
        self.bias = bias
        self.conv = nn.ConvTranspose2d(1, 1,
                                       kernel_size=(1, self.upsampling_factor),
                                       stride=(1, self.upsampling_factor),
                                       bias=self.bias)

    def forward(self, x):
        """x (B, C, T) -> (B, C, T * upsampling_factor)."""
        C = x.size(1)
        b = self.conv.bias if self.bias else torch.zeros(1, device=x.device)
        out = _UpsampleFn.apply(x, self.conv.weight, b, _round_up(C, 32))
        return out[:, :, :C].transpose(1, 2)


def _round_up(a, m):
    return (a + m - 1) // m * m


# ------------------------------------------------------------------------------------------
# resumable decoding (include/wnb200.h, wnb_decode_at): host arithmetic and the session object
# ------------------------------------------------------------------------------------------
DecodeWindow = collections.namedtuple("DecodeWindow", "pos0 end i0 n counts xs_base h_frame0")

# positions are int in the kernels: the last xs column written (P - 1 + the longest utterance) must stay below this
MAX_DECODE_POSITION = 2 ** 31 - 2


def decode_window(pos, frames, P, n_pad, U, ks, totals):
    """The next call of a resumable decode session: which positions it runs and the window arguments of wnb_decode_at.

    ``pos`` is the first padded position not yet run, ``frames`` the aux columns received so far (frames before
    up-sampling when U > 0, sample-rate columns when U == 0), ``P = max(T0, receptive_field)``, ``n_pad = P - T0``,
    ``totals`` the samples wanted per utterance.  Position p needs aux column ``max(p - n_pad, 0)``, i.e. frame
    ``max(p - n_pad, 0) // U``, so after ``frames`` frames the positions ``p < n_pad + frames * max(U, 1)`` can run.
    A call runs ``pos0 = pos`` up to ``end - 1`` and must generate at least one sample, so the P - 1 warm-up positions run
    in the first call that also reaches sample 0 (with a one-sample seed, the first call).  Returns None when no sample
    can be generated yet, else a DecodeWindow: ``i0`` the first sample index, ``n`` the samples of the longest utterance
    (max_n of the call), ``counts`` the samples per utterance (capped by ``totals``), ``xs_base`` the first xs column
    the call reads, ``h_frame0`` the first aux frame it reads."""
    Uc = max(U, 1)
    avail = n_pad + frames * Uc if frames > 0 else 0
    end = min(avail, P - 1 + max(totals))
    n = end - max(pos, P - 1)
    if n <= 0:
        return None
    i0 = max(pos - (P - 1), 0)
    counts = [min(max(t - i0, 0), n) for t in totals]
    return DecodeWindow(pos, end, i0, n, counts, max(pos - (ks - 1), 0), max(pos - n_pad, 0) // Uc)


def decode_prefill_windows(dilations, ks):
    """The pruned windows of the parallel warm-up (csrc/decode_prefill.cu): ``S[l] = (ks - 1) * sum(dilations[l:])``, the
    number of warm-up positions just before P - 1 on which layer l's input x_l is needed.  Layer l's queue holds its last
    (ks - 1) * d_l, and x_{l+1} on its own window needs x_l on taps up to (ks - 1) * d_l further back; x_L is never
    queued.  The library computes the same windows (``wnb_decode_prefill_windows``: the prefill launcher's ranges and the
scratch size of ``wnb_decode_prefill_workspace``); the CPU tier checks that both agree."""
    out, S = [], 0
    for d in reversed(dilations):
        S += (ks - 1) * d
        out.append(S)
    return out[::-1]


def _warp_prefill(lib, xs, P, h, upw, upb, w, dil, L, queues, n_pad, A, U, CL):
    """Run the warm-up positions 0 .. P - 2 of ``wnb_decode_warp_at`` in parallel over time (wnb_decode_warp_prefill):
    the queues then hold what the sequential warm-up leaves there, and ``wnb_decode_warp_at`` continues from P - 1."""
    B = xs.size(0)
    nbytes = lib.wnb_decode_prefill_workspace(B, P, 64, 2, dil, L)
    scratch = torch.empty(nbytes // 4, dtype=torch.float32, device=xs.device) if nbytes else None
    check(lib.wnb_decode_warp_prefill(ptr(xs[:, :P].contiguous()), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]),
                                      ptr(w["bf"]), ptr(w["w1d"]), ptr(w["b1"]), ptr(w["w2d"]), ptr(w["b2"]), dil, L,
                                      ptr(queues), ptr(scratch), B, P, n_pad, h.size(2), A, U, CL, stream()),
          "decode_warp_prefill")


def _decode_snapshot(net):
    """The decode weights a session or pool keeps for its whole life: ``_decode_pack()`` and the up-sampling weight and
    bias (None without an up-sampling layer).  Copies: ``_decode_pack()`` hands some entries (the front and post biases)
    out as the parameters themselves, and an in-place update of the model (load_state_dict, an optimizer step) must not
    reach a running decode."""
    params = {p.untyped_storage().data_ptr() for p in net.parameters()}
    w = {k: v.clone() if v.untyped_storage().data_ptr() in params else v for k, v in net._decode_pack().items()}
    U = net.upsampling_factor
    upw = net.upsampling.conv.weight.detach().float().contiguous().view(-1).clone() if U > 0 else None
    upb = net.upsampling.conv.bias.detach().float().contiguous().view(-1).clone() if U > 0 else None
    return w, upw, upb


def _bf16_weight_stream(lib, net):
    """The packed weight stream of the bf16 decoder (``_decode_bf16_pack``); raises for a shape it does not cover."""
    Q, A, Ap, R, S, ks, L = (net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size,
                             len(net.dilations))
    if not lib.wnb_decode_bf16_supported(Q, Ap, R, S, ks, L):
        raise _lib.WnbError("decode_math='bf16' does not cover this model (n_quantize %d, n_aux %d, n_resch %d, "
                            "n_skipch %d, kernel_size %d, %d layers): see decode_bf16_supported()" % (Q, A, R, S, ks, L))
    wstream = net._decode_bf16_pack()
    assert wstream.numel() == lib.wnb_decode_bf16_weights(Q, Ap, R, S, ks, L)
    return wstream


def _bf16_prefill(lib, xs, P, h, upw, upb, w, wstream, dil, L, queues, n_pad, A, Ap, R, S, ks, U):
    """Run the warm-up positions 0 .. P - 2 of the bf16 decoder in parallel over time (wnb_decode_bf16_prefill): the
    queues then hold what the sequential warm-up leaves there, and ``wnb_decode_bf16_at`` continues from P - 1."""
    B = xs.size(0)
    nbytes = lib.wnb_decode_bf16_prefill_workspace(B, P, R, ks, dil, L)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=xs.device) if nbytes else None
    check(lib.wnb_decode_bf16_prefill(ptr(xs[:, :P].contiguous()), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]),
                                      ptr(w["bf"]), ptr(wstream), dil, L, ptr(queues), ptr(scratch), B, P, n_pad,
                                      h.size(2), A, Ap, R, S, ks, U, stream()),
          "decode_bf16_prefill")


# utterances one streaming-decoder prefill launch sequence takes at most: the library groups larger batches, so the
# scratch stays at 2 * 64 * R * min(S_0, P - 1) floats
STREAM_PREFILL_ROWS = 64


def _stream_prefill(lib, xs, P, h, upw, upb, w, wstream, dil, L, queues, n_pad, Q, A, Ap, R, S, ks, U):
    """Run the warm-up positions 0 .. P - 2 of ``wnb_decode_stream_at`` in parallel over time
    (wnb_decode_stream_prefill): the queues then hold what the sequential warm-up leaves there, and
    ``wnb_decode_stream_at`` continues from P - 1."""
    B = xs.size(0)
    nbytes = lib.wnb_decode_prefill_workspace(min(B, STREAM_PREFILL_ROWS), P, R, ks, dil, L)
    scratch = torch.empty(nbytes // 4, dtype=torch.float32, device=xs.device) if nbytes else None
    check(lib.wnb_decode_stream_prefill(ptr(xs[:, :P].contiguous()), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]),
                                        ptr(w["bf"]), ptr(wstream), ptr(w["b1"]), ptr(w["b2"]), dil, L, ptr(queues),
                                        ptr(scratch), B, P, n_pad, h.size(2), Q, A, Ap, R, S, ks, U, stream()),
          "decode_stream_prefill")


class DecodeSession(object):
    """A resumable decode of a batch of utterances, fed with aux frames as they arrive (``WaveNet.decode_session``).

    This is the one place that picks a decoder and launches it: one-shot decoding (``WaveNet._decode``) is a session
    given every aux frame in its first call.  Each ``step(h_chunk)`` runs one launch of the decoder and returns the
    samples whose aux has now arrived; the chained calls compute exactly what ``batch_fast_generate`` computes for the
    same seed, whatever the chunk sizes.  Everything the calls share lives here, created once: the launch form, a snapshot
    of the packed weights (and of ``decode_math``), the dilation queues, the last ks - 1 samples and the seed.  All
    utterances advance together; utterance b stops at ``n_samples_list[b]``.

    ``kernel``: "auto" runs the bf16 decoder under ``decode_math="bf16"`` (an uncovered shape raises), and otherwise the
    warp-tiled decoder where it covers the shape, else the streaming one, else the direct one.  A named kernel ("warp",
    "stream", "direct", "bf16") runs that kernel or raises."""

    def __init__(self, net, x, n_samples_list, mode="sampling", seed=None, uniforms=None, return_logits=False,
                 kernel="auto"):
        if mode not in ("sampling", "argmax"):
            logging.error("mode should be sampling or argmax")
            sys.exit(1)
        if not x.is_cuda:
            raise _lib.WnbError("decode sessions need CUDA tensors: this build has no CPU fallback")
        lib = _lib.load()
        decode_math = getattr(net, "decode_math", "fp32")
        if decode_math not in ("fp32", "bf16"):
            raise ValueError("decode_math should be fp32 or bf16, got %r" % (decode_math,))
        if kernel not in ("auto", "warp", "stream", "direct", "bf16"):
            raise ValueError("unknown decode kernel %r" % (kernel,))
        if kernel == "auto" and decode_math == "bf16":
            kernel = "bf16"
        self.device = dev = x.device
        B, T0 = x.shape
        self.totals = [int(n) for n in n_samples_list]
        if len(self.totals) != B or min(self.totals) < 0:
            raise ValueError("n_samples_list should hold %d non-negative lengths, got %r" % (B, n_samples_list))
        self.Q, self.A, self.Ap, self.R, self.S, self.ks, self.U = (
            net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size, net.upsampling_factor)
        Q, Ap, R, S, ks, U = self.Q, self.Ap, self.R, self.S, self.ks, self.U
        self.B, self.P = B, max(T0, net.receptive_field)
        self.n_pad = self.P - T0
        if self.P - 1 + max(self.totals) > MAX_DECODE_POSITION:
            raise ValueError("a decode session covers at most %d positions (%d requested)"
                             % (MAX_DECODE_POSITION, self.P - 1 + max(self.totals)))
        L = len(net.dilations)
        self.L = L
        self.dil = (ctypes.c_int32 * L)(*net.dilations)
        self.mode = MODE_ARGMAX if mode == "argmax" else MODE_SAMPLING
        self.w, self.upw, self.upb = _decode_snapshot(net)
        if kernel == "bf16":
            self.wstream = _bf16_weight_stream(lib, net)
            qbytes = lib.wnb_decode_bf16_workspace(B, R, ks, self.dil, L)
        else:
            if kernel in ("auto", "warp"):
                if (lib.wnb_decode_warp_supported(Q, Ap, R, S, ks, L)
                        and lib.wnb_decode_warp_form(B, L, (ctypes.c_int32 * 4)()) == 0):
                    kernel = "warp"
                elif kernel == "warp":
                    raise _lib.WnbError("decode kernel 'warp' does not cover this configuration")
                else:
                    kernel = "stream" if lib.wnb_decode_stream_supported(Q, Ap, R, S, ks, L) else "direct"
            if kernel == "warp":
                self.W, self.CL = lib.wnb_decode_warp_plan(B), lib.wnb_decode_warp_cluster(B)
                self.wstream = net._decode_warp_pack(self.W, self.CL)
                assert self.wstream.numel() == lib.wnb_decode_warp_floats(L, self.CL)
            elif kernel == "stream":
                self.wstream = net._decode_stream_pack(self.w)
                assert self.wstream.numel() == lib.wnb_decode_stream_floats(Q, Ap, R, S, ks, L)
                # the parallel warm-up serves the models the streaming decoder runs by default, every fp32 shape outside
                # the warp decoder; on a shape the warp decoder covers, "stream" runs only when named, and stays the
                # one-launch sequential decode that cross-checks the other decoders
                self._parallel_warmup = not lib.wnb_decode_warp_supported(Q, Ap, R, S, ks, L)
            qbytes = lib.wnb_decode_workspace(B, R, ks, self.dil, L)
        self.kernel = kernel
        self.queues = torch.empty(max(qbytes // 4, 1), dtype=torch.float32, device=dev)
        if seed is None:
            seed = int(torch.empty((), dtype=torch.int64).random_().item())  # follows torch.manual_seed, like _decode
        self.seed = ctypes.c_uint64(seed & 0xFFFFFFFFFFFFFFFF)
        self.uniforms = None if uniforms is None else uniforms.to(dev).float().contiguous()
        self.return_logits = return_logits
        self._totals_dev = torch.tensor(self.totals, dtype=torch.int32, device=dev)
        # xs carry: the seed prefix first, then the last ks - 1 positions a call has written (absolute column _xs_base)
        self._xs = torch.full((B, self.P), Q // 2, dtype=torch.int32, device=dev)
        self._xs[:, self.n_pad:] = x.to(torch.int32)
        self._xs_base = 0
        # aux frames received and not yet behind every position run (absolute frame _h0 first)
        self._h = torch.empty(B, self.A, 0, dtype=torch.float32, device=dev)
        self._h0 = 0
        self.frames = 0
        self.pos = 0
        self.last_counts = [0] * B
        self._pcm_tab = None   # built by the first step_pcm16: it costs a launch and a synchronisation

    @property
    def done(self):
        """True once every utterance has all its samples."""
        return self.pos >= self.P - 1 + max(self.totals)

    def step(self, h_chunk):
        """Feed the next aux frames ``(B, n_aux, F)`` (sample-rate columns when the model has no up-sampling layer) and
        decode every position whose aux has now arrived.  Returns the new codes as a ``(B, n)`` int32 device tensor,
        without synchronising; row b holds ``last_counts[b]`` valid samples (an utterance past its length gets none).
        With ``return_logits`` the ``(B, n, Q)`` teacher-check logits come as a second value."""
        lib = _lib.load()
        if self.done:
            raise RuntimeError("decode session: every utterance has finished")
        if not h_chunk.is_cuda:
            raise _lib.WnbError("decode sessions need CUDA tensors: this build has no CPU fallback")
        if h_chunk.dim() != 3 or h_chunk.size(0) != self.B or h_chunk.size(1) != self.A:
            raise ValueError("aux chunk should be (%d, %d, frames), got %s" % (self.B, self.A, tuple(h_chunk.shape)))
        self._h = torch.cat([self._h, h_chunk.to(self.device).float()], 2)
        self.frames += h_chunk.size(2)
        win = decode_window(self.pos, self.frames, self.P, self.n_pad, self.U, self.ks, self.totals)
        B, Q = self.B, self.Q
        if win is None:
            self.last_counts = [0] * B
            gen = torch.empty(B, 0, dtype=torch.int32, device=self.device)
            return (gen, torch.empty(B, 0, Q, device=self.device)) if self.return_logits else gen
        h = self._h[:, :, win.h_frame0 - self._h0:].contiguous()
        xs = torch.full((B, win.end + 1 - win.xs_base), Q // 2, dtype=torch.int32, device=self.device)
        hi = min(self._xs_base + self._xs.size(1), win.end + 1)
        xs[:, :hi - win.xs_base] = self._xs[:, win.xs_base - self._xs_base:hi - self._xs_base]
        nsm = (self._totals_dev - win.i0).clamp_(0, win.n)
        uni = None if self.uniforms is None else self.uniforms[:, win.i0:win.i0 + win.n].contiguous()
        lg = torch.empty(B, win.n, Q, dtype=torch.float32, device=self.device) if self.return_logits else None
        w, st = self.w, stream()
        common = (B, self.P, win.n, self.n_pad, h.size(2))
        window = (win.pos0, win.xs_base, win.h_frame0, st)
        if self.kernel == "bf16":
            if win.pos0 == 0:   # the warm-up in parallel over time, then this call from P - 1 (xs and h start at 0)
                _bf16_prefill(lib, xs, self.P, h, self.upw, self.upb, w, self.wstream, self.dil, self.L, self.queues,
                              self.n_pad, self.A, self.Ap, self.R, self.S, self.ks, self.U)
                window = (self.P - 1, 0, 0, st)
            rc = lib.wnb_decode_bf16_at(ptr(xs), ptr(h), ptr(self.upw), ptr(self.upb), ptr(w["wf"]), ptr(w["bf"]),
                                        ptr(self.wstream), self.dil, self.L, ptr(self.queues), ptr(nsm), ptr(uni), ptr(lg),
                                        *common, Q, self.A, self.Ap, self.R, self.S, self.ks, self.U, self.mode, self.seed,
                                        *window)
        elif self.kernel == "warp":
            if win.pos0 == 0:   # the warm-up in parallel over time, then this call from P - 1 (xs and h start at 0)
                _warp_prefill(lib, xs, self.P, h, self.upw, self.upb, w, self.dil, self.L, self.queues, self.n_pad,
                              self.A, self.U, self.CL)
                window = (self.P - 1, 0, 0, st)
            rc = lib.wnb_decode_warp_at(ptr(xs), ptr(h), ptr(self.upw), ptr(self.upb), ptr(w["wf"]), ptr(w["bf"]),
                                        ptr(self.wstream), ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]),
                                        self.dil, self.L, ptr(self.queues), ptr(nsm), ptr(uni), ptr(lg), *common, self.A,
                                        self.U, self.mode, self.seed, self.W, self.CL, *window)
        elif self.kernel == "stream":
            if win.pos0 == 0 and self._parallel_warmup:   # the warm-up in parallel over time, then this call from P - 1
                _stream_prefill(lib, xs, self.P, h, self.upw, self.upb, w, self.wstream, self.dil, self.L, self.queues,
                                self.n_pad, Q, self.A, self.Ap, self.R, self.S, self.ks, self.U)
                window = (self.P - 1, 0, 0, st)
            rc = lib.wnb_decode_stream_at(ptr(xs), ptr(h), ptr(self.upw), ptr(self.upb), ptr(w["wf"]), ptr(w["bf"]),
                                          ptr(self.wstream), ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]),
                                          self.dil, self.L, ptr(self.queues), ptr(nsm), ptr(uni), ptr(lg), *common, Q,
                                          self.A, self.Ap, self.R, self.S, self.ks, self.U, self.mode, self.seed, *window)
        else:
            rc = lib.wnb_decode_at(ptr(xs), ptr(h), ptr(self.upw), ptr(self.upb), ptr(w["wf"]), ptr(w["bf"]),
                                   ptr(w["w1d"]), ptr(w["b1"]), ptr(w["w2d"]), ptr(w["b2"]), ptr(w["wp1d"]),
                                   ptr(w["bp1"]), ptr(w["wp2d"]), ptr(w["bp2"]), self.dil, self.L, ptr(self.queues),
                                   ptr(nsm), ptr(uni), ptr(lg), *common, Q, self.A, self.Ap, self.R, self.S, self.ks,
                                   self.U, self.mode, self.seed, *window)
        check(rc, "decode_%s_at" % self.kernel)
        self._xs, self._xs_base = xs, win.xs_base
        self.pos = win.end
        f = max(self.pos - self.n_pad, 0) // max(self.U, 1)   # frames before the next position are no longer needed
        self._h, self._h0 = self._h[:, :, f - self._h0:], f
        self.last_counts = win.counts
        gen = xs[:, self.P + win.i0 - win.xs_base:self.P + win.i0 + win.n - win.xs_base]
        return (gen, lg) if self.return_logits else gen

    def step_pcm16(self, h_chunk):
        """``step`` with the new samples as PCM_16 (``decode_mu_law`` + the wav writer's quantisation, one gather
        kernel): a ``(B, n)`` int16 device tensor, without synchronising after the first call."""
        if self._pcm_tab is None:
            self._pcm_tab = torch.from_numpy(mulaw_pcm16_table(self.Q)).to(self.device)
        gen = self.step(h_chunk)
        codes = (gen[0] if self.return_logits else gen).contiguous()
        out = torch.empty(codes.shape, dtype=torch.int16, device=self.device)
        check(_lib.load().wnb_lut_i16(ptr(codes), ptr(self._pcm_tab), ptr(out), codes.numel(), self.Q, stream()),
              "lut_i16")
        return out


# A decode pool's global step counter g is a decoder position: it stays at or below this (the last position of a call,
# g0 + n).  Before a call would pass it, g drops by a multiple of every queue length, which leaves every slot in place.
POOL_COUNTER_LIMIT = MAX_DECODE_POSITION
# steps of one pool call at most: the call's aux window is staged at sample rate, (capacity, n_aux, n) fp32
POOL_MAX_STEPS = 8192
# streams one admission prefill takes at most: one cluster of the bf16 decoder
POOL_ADMIT_ROWS = 64

PoolCall = collections.namedtuple("PoolCall", "g0 n admit rows finished park resume")


class PoolStream(object):
    """One stream of a decode pool: seed length T0 (P = max(T0, rf), n_pad = P - T0), length, aux frames received,
    samples decoded and the pool slot it occupies (None while it waits or is parked)."""

    def __init__(self, sid, T0, total, rf):
        self.sid, self.T0, self.total = sid, T0, total
        self.P = max(T0, rf)
        self.n_pad = self.P - T0
        self.frames, self.done, self.slot = 0, 0, None

    def runnable(self, U, ks):
        """Samples after the decoded ones whose aux has arrived (``decode_window``'s rule)."""
        win = decode_window(self.P - 1 + self.done, self.frames, self.P, self.n_pad, U, ks, [self.total])
        return win.n if win is not None else 0

    def aux_column(self, i):
        """The aux column (sample rate) of sample i: position P - 1 + i less the n_pad replicated columns."""
        return self.T0 - 1 + i

    @property
    def position(self):
        """The stream's next decoder position: P - 1 + samples decoded."""
        return self.P - 1 + self.done


class PoolSchedule(object):
    """The host arithmetic of a ``DecodePool``, with no device work: which streams enter which slots, how many steps a
    call runs and which samples every row makes.  ``next_call`` applies the rules of ``DecodePool.step`` and returns a
    ``PoolCall``, or None when no stream can run:
      * ``g0``, ``n``: the call runs the pool's steps g0 .. g0 + n - 1;
      * ``admit``: groups ``(T0, [stream, ...])`` of at most POOL_ADMIT_ROWS streams with one seed length, each one
        prefill; a stream's queue slots rotate by ``g0 - (P - 1)`` (its first sample is step g0);
      * ``rows``: ``(slot, stream, i0, count)`` for every occupied slot: samples i0 .. i0 + count - 1;
      * ``finished``: the ids of the streams this call completes (their slots are free for the next call);
      * ``park``: ``(slot, stream, rotation)`` for every stream that leaves its slot for a store before the call;
        ``rotation = v - g0`` for its next position v (the store's slot s holds position v' = s mod qlen);
      * ``resume``: ``(slot, stream, rotation)`` for every parked stream that enters a free slot after the admissions;
        ``rotation = g0 - v`` (its next sample is step g0).

    ``park_below=None`` is lock step: every stream in a slot stays there until it finishes, and a stream whose aux has not
    arrived bounds the whole call.  With ``park_below=m`` (an int >= 1), a stream needs ``min(m, samples left)``
    runnable samples to hold a slot: a stream in a slot with fewer is parked, and a parked stream that has them again is
    resumed into any free slot, ahead of the waiting streams.  A stream whose aux is complete is never parked.

    ``g_base`` is the lowest step counter (default ks - 1: the front gather reads g - (ks - 1) .. g, never a position
    below 0); the counter starts there and a rebase stays at or above it."""

    def __init__(self, capacity, receptive_field, dilations, ks, U, park_below=None, g_base=None):
        if park_below is not None and (not isinstance(park_below, int) or park_below < 1):
            raise ValueError("park_below should be None or an int >= 1, got %r" % (park_below,))
        self.capacity, self.rf, self.ks, self.U = capacity, receptive_field, ks, U
        self.park_below = park_below
        self.period = 1                      # lcm of the queue lengths (ks - 1) d_l
        for d in dilations:
            q = (ks - 1) * d
            self.period = self.period * q // math.gcd(self.period, q)
        self.g_base = ks - 1 if g_base is None else int(g_base)
        if self.g_base < ks - 1:
            raise ValueError("g_base should be at least ks - 1 = %d, got %d" % (ks - 1, self.g_base))
        self.g = self.g_base
        self.slots = [None] * capacity
        self.waiting = []                    # FIFO
        self.parked = []                     # in the order they were parked
        self.streams = {}                    # id -> PoolStream, until it finishes or is cancelled
        self.finished = set()                # ids of the streams that finished or were cancelled

    def add(self, sid, T0, total):
        st = PoolStream(sid, T0, total, self.rf)
        self.streams[sid] = st
        self.waiting.append(st)
        return st

    def cancel(self, sid):
        """Remove a waiting, active or parked stream; an active stream's slot is free for the next call."""
        st = self.streams.pop(sid)
        if st in self.waiting:
            self.waiting.remove(st)
        elif st in self.parked:
            self.parked.remove(st)
        else:
            self.slots[st.slot] = None
        st.slot = None
        self.finished.add(sid)
        return st

    def _fits(self, st):
        """Under park_below: the stream can run the samples it needs to hold a slot."""
        return st.runnable(self.U, self.ks) >= min(self.park_below, st.total - st.done)

    def next_call(self, max_samples=None):
        U, ks = self.U, self.ks
        # the plan works on a copy: a call that launches nothing changes nothing
        slots, park, resume = list(self.slots), [], []
        if self.park_below is None:
            free = [s for s, st in enumerate(slots) if st is None]
            ready = [st for st in self.waiting if st.runnable(U, ks) > 0][:len(free)]
        else:
            for s, st in enumerate(slots):
                if st is not None and not self._fits(st):
                    park.append((s, st))
                    slots[s] = None
            free = [s for s, st in enumerate(slots) if st is None]
            resume = [st for st in self.parked if self._fits(st)][:len(free)]
            ready = [st for st in self.waiting if self._fits(st)][:len(free) - len(resume)]
        active = [st for st in slots if st is not None] + resume + ready
        if not active:
            return None
        # one launch for every row: a stream whose aux is still incomplete bounds the call by what it can run
        n = max(st.total - st.done for st in active)
        for st in active:
            r = st.runnable(U, ks)
            if r < st.total - st.done:
                n = min(n, r)
        n = min(n, POOL_MAX_STEPS if max_samples is None else min(max_samples, POOL_MAX_STEPS))
        if n <= 0:
            return None
        if self.g + n > POOL_COUNTER_LIMIT:
            self.g = self.g_base + (self.g - self.g_base) % self.period
            if self.g >= POOL_COUNTER_LIMIT:
                raise ValueError("POOL_COUNTER_LIMIT %d leaves no step after a rebase to %d"
                                 % (POOL_COUNTER_LIMIT, self.g))
            n = min(n, POOL_COUNTER_LIMIT - self.g)
        # rotations from g0: a rebase moves g by a multiple of every queue length, so a parked row's slots do not care
        park_calls, resume_calls = [], []
        for s, st in park:
            park_calls.append((s, st, st.position - self.g))
            self.slots[s], st.slot = None, None
            self.parked.append(st)
        free = iter(free)
        for st in resume:
            s = next(free)
            resume_calls.append((s, st, self.g - st.position))
            self.parked.remove(st)
            st.slot, self.slots[s] = s, st
        groups = collections.OrderedDict()
        for st, s in zip(ready, free):
            self.waiting.remove(st)
            st.slot, self.slots[s] = s, st
            groups.setdefault(st.T0, []).append(st)
        admit = [(T0, sts[k:k + POOL_ADMIT_ROWS]) for T0, sts in groups.items()
                 for k in range(0, len(sts), POOL_ADMIT_ROWS)]
        rows, finished = [], []
        for s, st in enumerate(self.slots):
            if st is None:
                continue
            c = min(st.total - st.done, n)
            rows.append((s, st, st.done, c))
            st.done += c
            if st.done == st.total:
                finished.append(st.sid)
                self.slots[s] = None          # (st.slot keeps the row: this call's admission still needs it)
                del self.streams[st.sid]
                self.finished.add(st.sid)
        g0 = self.g
        self.g += n
        return PoolCall(g0, n, admit, rows, finished, park_calls, resume_calls)


def warp_pool_supported(net, capacity):
    """True when the fp32 warp decoder covers ``net`` at a pool of ``capacity`` rows (``warp_pool_form`` would not
    raise)."""
    lib = _lib.load()
    Q, Ap, R, S, ks, L = (net.n_quantize, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size, len(net.dilations))
    return bool(lib.wnb_decode_warp_supported(Q, Ap, R, S, ks, L)
                and lib.wnb_decode_warp_form(capacity, L, (ctypes.c_int32 * 4)()) == 0)


def warp_pool_form(net, capacity):
    """(NU, W, CL): the form ``wnb_decode_warp_at`` runs for a pool of ``capacity`` rows on the fp32 warp decoder
    (``wnb_decode_warp_form``).  The thresholds are the library's and follow the device's SM count: on a 132-SM H100 one
    utterance per 2-CTA cluster up to 66 rows, one per CTA up to 132, two up to 264, four beyond.  Raises ``WnbError``
    for a model or capacity the warp decoder does not cover."""
    lib = _lib.load()
    Q, A, Ap, R, S, ks, L = (net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size,
                             len(net.dilations))
    form = (ctypes.c_int32 * 4)()
    if not lib.wnb_decode_warp_supported(Q, Ap, R, S, ks, L) or lib.wnb_decode_warp_form(capacity, L, form) != 0:
        raise _lib.WnbError("decode_math='fp32' pools run the warp decoder, which does not cover this model (n_quantize "
                            "%d, n_aux %d, n_resch %d, n_skipch %d, kernel_size %d, %d layers) at capacity %d: it covers "
                            "n_quantize 256, n_aux <= 32, n_resch 64, n_skipch 512, kernel_size 2; decode_math='bf16' "
                            "pools cover the recipe sizes, and kernel='stream' runs an fp32 pool on the streaming "
                            "decoder" % (Q, A, R, S, ks, L, capacity))
    return form[0], form[1], form[2]


def pool_kernel(decode_math, kernel):
    """The decoder a ``DecodePool`` runs: "auto" is "bf16" under ``decode_math="bf16"`` and "warp" under "fp32"; a named
    kernel must belong to the pool's math ("bf16" to bf16, "warp" and "stream" to fp32).  Raises ``WnbError``
    otherwise."""
    if decode_math not in ("fp32", "bf16"):
        raise _lib.WnbError("decode pools run the bf16 decoder (decode_math='bf16') or an fp32 decoder "
                            "(decode_math='fp32'), got %r" % (decode_math,))
    if kernel == "auto":
        return "bf16" if decode_math == "bf16" else "warp"
    if kernel not in ("warp", "stream", "bf16"):
        raise ValueError("unknown decode pool kernel %r: 'auto', 'warp', 'stream' or 'bf16'" % (kernel,))
    if (kernel == "bf16") != (decode_math == "bf16"):
        raise _lib.WnbError("decode pool kernel %r does not run decode_math=%r" % (kernel, decode_math))
    return kernel


def _pinned_int32(values, dev):
    """A host list as an int32 device tensor, copied without synchronising the host (pinned staging)."""
    return torch.tensor(values, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)


class DecodePool(object):
    """Continuous batching (``WaveNet.decode_pool``): streams join a free row of a running batch and leave it the moment
    they finish, so requests that arrive at different times share one weight read.  Under ``decode_math="bf16"`` the
    pool runs the bf16 decoder, under "fp32" the fp32 warp decoder (``warp_pool_form``: the BASELINE shape, 64 res /
    512 skip, ks 2; another shape raises ``WnbError``), or with ``kernel="stream"`` the fp32 streaming decoder, which
    covers every shape ``wnb_decode_stream_supported`` accepts (``pool_kernel``).

    The pool is one decoder batch of ``capacity`` rows (``wnb_decode_bf16_at`` or ``wnb_decode_warp_at``), launched once
    per ``step`` over the pool's global steps g0 .. g0 + n - 1 with P = 1, n_pad = 0, U = 0 (include/wnb200.h, DESIGN
    §3.7).  A stream's warm-up runs as the usual parallel prefill when it is admitted, and its queues are moved into its
    row, rotated so that its first sample is the pool's step of admission (``wnb_decode_bf16_pool_transplant``, or
    ``wnb_decode_pool_move`` on the warp decoder, whose prefill runs with the pool's CL); each call's aux window and
    uniforms are written per row for the row's own stream (``wnb_decode_bf16_pool_inputs``, shared by both decoders).
    Stream k of a bf16 pool with seed S decodes exactly what row k of ``net._decode(X, H, n_list, mode, seed=S,
    kernel="bf16")`` decodes, bit for bit.  Stream k of an fp32 pool with seed S decodes what row k of
    ``net._decode(X, H, n_list, mode, seed=S, kernel="warp")`` decodes, bit for bit, for a one-shot batch whose warp form
    (``wnb_decode_warp_form``: NU, W, CL) equals the pool's: the form sets the order of some fp32 sums.  On
    ``kernel="stream"`` (admission: ``wnb_decode_stream_prefill`` and ``wnb_decode_pool_move``) stream k equals row k of
    ``net._decode(X, H, n_list, mode, seed=S, kernel="stream")`` for any one-shot batch size: the streaming decoder's sums
    do not depend on its launch form.

    ``step`` runs one launch for every row.  By default (``park_below=None``) it advances in lock step: a stream whose
    aux frames have not arrived holds back the whole launch (the call runs only what that stream can run, and nothing if
    it can run nothing).  That suits a local acoustic model, which stays ahead of the bf16 decoder (about 1.6 k samples/s
    per stream at arctic 512/256).  With ``park_below=m``, a stream that cannot run ``min(m, samples left)`` samples is
    parked instead: its queues move out of its row into a store of its own (``wnb_decode_bf16_pool_park``, or
    ``wnb_decode_pool_move`` on the warp decoder), its row serves other streams, and once its frames arrive it is
    resumed into any free row (``wnb_decode_bf16_pool_unpark``, or ``wnb_decode_pool_move``),
    ahead of the waiting streams, with the same codes.  ``m = 1`` parks only streams that can run nothing; a larger m
    keeps a slow stream from cutting every call short.  ``cancel`` drops a stream at once.  The pool snapshots the
    weights at its creation."""

    def __init__(self, net, capacity=64, mode="sampling", seed=None, park_below=None, kernel="auto"):
        if mode not in ("sampling", "argmax"):
            raise ValueError("mode should be sampling or argmax, got %r" % (mode,))
        capacity = int(capacity)
        if capacity < 1:
            raise ValueError("a decode pool needs a capacity of at least 1, got %d" % capacity)
        kernel = pool_kernel(getattr(net, "decode_math", "fp32"), kernel)
        lib = _lib.load()
        self.device = dev = _device()
        self.Q, self.A, self.Ap, self.R, self.S, self.ks, self.U = (
            net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size, net.upsampling_factor)
        self.rf, self.L, self.capacity = net.receptive_field, len(net.dilations), capacity
        self.dil = (ctypes.c_int32 * self.L)(*net.dilations)
        self.kernel = kernel
        self.w, self.upw, self.upb = _decode_snapshot(net)
        g_base = None
        if self.kernel == "bf16":
            self.wstream = _bf16_weight_stream(lib, net)
            qbytes = lib.wnb_decode_bf16_workspace(capacity, self.R, self.ks, self.dil, self.L)
            admit_bytes = lib.wnb_decode_bf16_workspace(POOL_ADMIT_ROWS, self.R, self.ks, self.dil, self.L)
            self._park_bytes = lib.wnb_decode_bf16_park_bytes(self.R, self.ks, self.dil, self.L)
        else:
            if self.kernel == "warp":
                _, self.W, self.CL = warp_pool_form(net, capacity)
                self.wstream = net._decode_warp_pack(self.W, self.CL)
                assert self.wstream.numel() == lib.wnb_decode_warp_floats(self.L, self.CL)
            else:
                if not lib.wnb_decode_stream_supported(self.Q, self.Ap, self.R, self.S, self.ks, self.L):
                    raise _lib.WnbError("kernel='stream' pools run the streaming decoder, which does not cover this "
                                        "model (n_quantize %d, n_aux %d, n_resch %d, n_skipch %d, kernel_size %d, %d "
                                        "layers)" % (self.Q, self.A, self.R, self.S, self.ks, self.L))
                self.wstream = net._decode_stream_pack(self.w)
                assert self.wstream.numel() == lib.wnb_decode_stream_floats(self.Q, self.Ap, self.R, self.S, self.ks,
                                                                            self.L)
            # one utterance's queue block: a pool row, a row of the admission workspace and a parked stream's store
            self._block = lib.wnb_decode_workspace(1, self.R, self.ks, self.dil, self.L)
            qbytes, admit_bytes, self._park_bytes = capacity * self._block, POOL_ADMIT_ROWS * self._block, self._block
            # the fp32 decoders read layer l's tap only at positions >= d_l (a zero before): keep g at or above that
            g_base = (self.ks - 1) * max(net.dilations)
        self.mode = MODE_ARGMAX if mode == "argmax" else MODE_SAMPLING
        if seed is None:
            seed = int(torch.empty((), dtype=torch.int64).random_().item())  # follows torch.manual_seed, like _decode
        self.seed = ctypes.c_uint64(seed & 0xFFFFFFFFFFFFFFFF)
        # zeroed once: the decoder is never launched with pos0 = 0 here, so it never clears them
        self.queues = torch.zeros(qbytes, dtype=torch.uint8, device=dev)
        self._admit_queues = torch.empty(admit_bytes, dtype=torch.uint8, device=dev)
        self._tail = torch.full((capacity, self.ks), self.Q // 2, dtype=torch.int32, device=dev)   # xs at g - ks + 1 .. g
        self._sched = PoolSchedule(capacity, self.rf, net.dilations, self.ks, self.U, park_below, g_base)
        self._x = {}        # id -> seed codes, until admitted
        self._h = {}        # id -> [aux frames (A, F) on the device, absolute frame of column 0]
        self._parked = {}   # id -> (queue store, last ks codes), while parked
        self._admitted = 0
        self._pcm_tab = None

    @property
    def active(self):
        """Ids of the streams in the pool's rows, by row."""
        return [st.sid for st in self._sched.slots if st is not None]

    @property
    def waiting(self):
        """Ids of the admitted streams that wait for a row (or for the aux frames of their first sample), in order."""
        return [st.sid for st in self._sched.waiting]

    @property
    def parked(self):
        """Ids of the parked streams, in the order they were parked."""
        return [st.sid for st in self._sched.parked]

    def cancel(self, stream):
        """End ``stream`` at once, whether it waits, runs in a row (the row is free for the next call) or is parked.
        Codes ``step`` returned before stay valid; afterwards ``finished(stream)`` is True, ``feed`` raises KeyError and
        the id cannot be admitted again."""
        if stream not in self._sched.streams:
            raise KeyError("decode pool: unknown or finished stream %r" % (stream,))
        self._sched.cancel(stream)
        for d in (self._x, self._h, self._parked):
            d.pop(stream, None)

    def finished(self, stream):
        """True once every sample of ``stream`` has been returned by ``step``, or once it was cancelled."""
        if stream in self._sched.finished:
            return True
        if stream not in self._sched.streams:
            raise KeyError("decode pool: unknown stream %r" % (stream,))
        return False

    def admit(self, x, n_samples, h=None, stream=None):
        """Queue a stream with seed codes ``x`` (1-D, on the GPU) and ``n_samples`` samples to decode, optionally with
        its first aux frames ``h`` (n_aux, F).  Returns its id: ``stream``, or by default the number of streams admitted
        before it.  The id is the stream's Philox counter word, as the batch index is in one-shot decoding."""
        if not x.is_cuda or (h is not None and not h.is_cuda):
            raise _lib.WnbError("decode pools need CUDA tensors: this build has no CPU fallback")
        if x.dim() != 1 or x.numel() < 1:
            raise ValueError("seed codes should be a non-empty 1-D tensor, got shape %s" % (tuple(x.shape),))
        sid = self._admitted if stream is None else stream
        if not isinstance(sid, int) or not 0 <= sid < 2 ** 31:
            raise ValueError("stream ids are ints in [0, 2^31), got %r" % (sid,))
        if sid in self._sched.streams or sid in self._sched.finished:
            raise ValueError("decode pool: stream %d exists already" % sid)
        n_samples = int(n_samples)
        P = max(x.numel(), self.rf)
        if n_samples < 1 or P - 1 + n_samples > MAX_DECODE_POSITION:
            raise ValueError("a stream decodes 1 .. %d samples, got %d" % (MAX_DECODE_POSITION - (P - 1), n_samples))
        self._admitted += 1
        self._sched.add(sid, x.numel(), n_samples)
        self._x[sid] = x.to(torch.int32)
        self._h[sid] = [torch.empty(self.A, 0, dtype=torch.float32, device=self.device), 0]
        if h is not None:
            self.feed(sid, h)
        return sid

    def feed(self, stream, h_chunk):
        """Append aux frames ``h_chunk`` (n_aux, F) to ``stream`` (sample-rate columns when the model has no
        up-sampling layer)."""
        st = self._sched.streams.get(stream)
        if st is None:
            raise KeyError("decode pool: unknown or finished stream %r" % (stream,))
        if not h_chunk.is_cuda:
            raise _lib.WnbError("decode pools need CUDA tensors: this build has no CPU fallback")
        if h_chunk.dim() != 2 or h_chunk.size(0) != self.A:
            raise ValueError("aux chunk should be (%d, frames), got %s" % (self.A, tuple(h_chunk.shape)))
        buf = self._h[stream]
        buf[0] = torch.cat([buf[0], h_chunk.to(self.device).float()], 1)
        st.frames += h_chunk.size(1)

    def step(self, max_samples=None):
        """Admit the waiting streams whose first aux frames have arrived and run one launch of at most ``max_samples``
        steps.  Returns ``{stream: new codes}`` (int32 device tensors, without synchronising) for every stream in a row;
        ``{}`` and no launch when no stream can run.  In lock step the launch runs only as many steps as the least-fed
        stream in a row can run.  With ``park_below`` the call first parks the streams that cannot keep up, then admits
        waiting streams and resumes parked ones into the free rows (parked ones first), then runs the launch."""
        call, gen = self._call(max_samples)
        return {} if call is None else {st.sid: gen[slot, :c] for slot, st, _, c in call.rows}

    def step_pcm16(self, max_samples=None):
        """``step`` with the new samples as PCM_16 (one ``wnb_lut_i16`` gather for the whole call): int16 device
        tensors, without synchronising after the first call."""
        call, gen = self._call(max_samples)
        if call is None:
            return {}
        if self._pcm_tab is None:
            self._pcm_tab = torch.from_numpy(mulaw_pcm16_table(self.Q)).to(self.device)
        codes = gen.contiguous()
        out = torch.empty(codes.shape, dtype=torch.int16, device=self.device)
        check(_lib.load().wnb_lut_i16(ptr(codes), ptr(self._pcm_tab), ptr(out), codes.numel(), self.Q, stream()),
              "lut_i16")
        return {st.sid: out[slot, :c] for slot, st, _, c in call.rows}

    def _admit_group(self, lib, T0, group, g0):
        """Prefill a group of streams with one seed length and move their queues into their rows."""
        P = max(T0, self.rf)
        n_pad, Bg, ks = P - T0, len(group), self.ks
        xs = torch.full((Bg, P), self.Q // 2, dtype=torch.int32, device=self.device)
        xs[:, n_pad:] = torch.stack([self._x.pop(st.sid) for st in group])
        Fg = min(self._h[st.sid][0].size(1) for st in group)
        h = torch.stack([self._h[st.sid][0][:, :Fg] for st in group]).contiguous()
        if self.kernel != "bf16":
            if self.kernel == "warp":
                # the pool's CL, not the group's: the 2-CTA form sums half of the residual products in another order
                _warp_prefill(lib, xs, P, h, self.upw, self.upb, self.w, self.dil, self.L, self._admit_queues, n_pad,
                              self.A, self.U, self.CL)
            else:
                _stream_prefill(lib, xs, P, h, self.upw, self.upb, self.w, self.wstream, self.dil, self.L,
                                self._admit_queues, n_pad, self.Q, self.A, self.Ap, self.R, self.S, ks, self.U)
            base = ptr(self._admit_queues)
            self._move(lib, [(base + k * self._block, self._row(st.slot), g0 - (P - 1)) for k, st in enumerate(group)])
            for k, st in enumerate(group):
                self._tail[st.slot] = xs[k, P - ks:]
            return
        _bf16_prefill(lib, xs, P, h, self.upw, self.upb, self.w, self.wstream, self.dil, self.L, self._admit_queues,
                      n_pad, self.A, self.Ap, self.R, self.S, ks, self.U)
        check(lib.wnb_decode_bf16_pool_transplant(ptr(self._admit_queues), Bg, (ctypes.c_int32 * Bg)(*range(Bg)),
                                                  ptr(self.queues), self.capacity,
                                                  (ctypes.c_int32 * Bg)(*[st.slot for st in group]),
                                                  (ctypes.c_int32 * Bg)(*[g0 - (P - 1)] * Bg), Bg, self.R, ks, self.dil,
                                                  self.L, stream()),
              "decode_bf16_pool_transplant")
        for k, st in enumerate(group):
            self._tail[st.slot] = xs[k, P - ks:]

    def _park(self, lib, park):
        """Copy the parked streams' rows into stores of their own (one launch per POOL_ADMIT_ROWS streams) and keep their
        last ks codes.  An active stream that has not finished ran every step of the last call, so its tail row ends at
        its last sample."""
        stores = [torch.empty(self._park_bytes, dtype=torch.uint8, device=self.device) for _ in park]
        if self.kernel != "bf16":
            self._move(lib, [(self._row(s), ptr(q), r) for (s, _, r), q in zip(park, stores)])
        else:
            self._bf16_park(lib, park, stores)
        tails = self._tail.index_select(0, _pinned_int32([s for s, _, _ in park], self.device).long())
        for k, (_, st, _) in enumerate(park):
            self._parked[st.sid] = (stores[k], tails[k])

    def _bf16_park(self, lib, park, stores):
        for k0 in range(0, len(park), POOL_ADMIT_ROWS):
            part = park[k0:k0 + POOL_ADMIT_ROWS]
            n = len(part)
            check(lib.wnb_decode_bf16_pool_park(ptr(self.queues), self.capacity, (ctypes.c_int32 * n)(*[s for s, _, _ in part]),
                                                (ctypes.c_void_p * n)(*[ptr(t) for t in stores[k0:k0 + n]]),
                                                (ctypes.c_int32 * n)(*[r for _, _, r in part]), n, self.R, self.ks,
                                                self.dil, self.L, stream()),
                  "decode_bf16_pool_park")

    def _unpark(self, lib, resume):
        """Copy the resumed streams' stores into their new rows (one launch per POOL_ADMIT_ROWS streams) and restore
        their last ks codes."""
        kept = [self._parked.pop(st.sid) for _, st, _ in resume]
        if self.kernel != "bf16":
            self._move(lib, [(ptr(q), self._row(s), r) for (s, _, r), (q, _) in zip(resume, kept)])
        else:
            self._bf16_unpark(lib, resume, kept)
        self._tail.index_copy_(0, _pinned_int32([s for s, _, _ in resume], self.device).long(),
                               torch.stack([t for _, t in kept]))

    def _bf16_unpark(self, lib, resume, kept):
        for k0 in range(0, len(resume), POOL_ADMIT_ROWS):
            part = resume[k0:k0 + POOL_ADMIT_ROWS]
            n = len(part)
            check(lib.wnb_decode_bf16_pool_unpark((ctypes.c_void_p * n)(*[ptr(q) for q, _ in kept[k0:k0 + n]]),
                                                  ptr(self.queues), self.capacity,
                                                  (ctypes.c_int32 * n)(*[s for s, _, _ in part]),
                                                  (ctypes.c_int32 * n)(*[r for _, _, r in part]), n, self.R, self.ks,
                                                  self.dil, self.L, stream()),
                  "decode_bf16_pool_unpark")

    def _row(self, slot):
        """Device address of pool row ``slot``'s queue block (fp32 pool)."""
        return ptr(self.queues) + slot * self._block

    def _move(self, lib, moves):
        """``wnb_decode_pool_move`` of ``(src, dst, rotation)`` queue blocks, one launch per POOL_ADMIT_ROWS moves."""
        for k0 in range(0, len(moves), POOL_ADMIT_ROWS):
            part = moves[k0:k0 + POOL_ADMIT_ROWS]
            n = len(part)
            check(lib.wnb_decode_pool_move((ctypes.c_void_p * n)(*[s for s, _, _ in part]),
                                           (ctypes.c_void_p * n)(*[d for _, d, _ in part]),
                                           (ctypes.c_int32 * n)(*[r for _, _, r in part]), n, self.R, self.ks, self.dil,
                                           self.L, stream()),
                  "decode_pool_move")

    def _call(self, max_samples):
        """One pool call: (PoolCall, (capacity, n) int32 codes of steps g0 .. g0 + n - 1), or (None, None)."""
        if max_samples is not None and int(max_samples) < 1:
            raise ValueError("max_samples should be at least 1, got %r" % (max_samples,))
        call = self._sched.next_call(max_samples)
        if call is None:
            return None, None
        lib = _lib.load()
        C, A, ks, Uc, n = self.capacity, self.A, self.ks, max(self.U, 1), call.n
        # parking first: a row it frees may take an admitted or a resumed stream in this same call
        if call.park:
            self._park(lib, call.park)
        for T0, group in call.admit:
            self._admit_group(lib, T0, group, call.g0)
        if call.resume:
            self._unpark(lib, call.resume)
        # each row's frames from the one of its first step, and the table of wnb_decode_bf16_pool_inputs
        table = [[0] * C for _ in range(5)]
        spans = []
        for slot, st, i0, c in call.rows:
            j0 = st.aux_column(i0)
            f0, f1 = j0 // Uc, (j0 + c - 1) // Uc + 1
            spans.append((slot, st, f0, f1))
            for r, v in enumerate((f0, j0, i0, st.sid, c)):
                table[r][slot] = v
        frames = torch.empty(C, A, max(f1 - f0 for _, _, f0, f1 in spans), dtype=torch.float32, device=self.device)
        for slot, st, f0, f1 in spans:
            buf, h0 = self._h[st.sid]
            frames[slot, :, :f1 - f0] = buf[:, f0 - h0:f1 - h0]
        tab = _pinned_int32(table, self.device)
        aux = torch.empty(C, A, n, dtype=torch.float32, device=self.device)
        uni = torch.empty(C, n, dtype=torch.float32, device=self.device) if self.mode == MODE_SAMPLING else None
        st_ = stream()
        check(lib.wnb_decode_bf16_pool_inputs(ptr(frames), ptr(self.upw), ptr(self.upb), ptr(tab), ptr(aux), ptr(uni), C,
                                              A, frames.size(2), n, self.U, self.seed, st_),
              "decode_bf16_pool_inputs")
        xs = torch.empty(C, ks + n, dtype=torch.int32, device=self.device)
        xs[:, :ks] = self._tail
        w, g0 = self.w, call.g0
        if self.kernel == "warp":
            check(lib.wnb_decode_warp_at(ptr(xs), ptr(aux), None, None, ptr(w["wf"]), ptr(w["bf"]), ptr(self.wstream),
                                         ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]), self.dil, self.L,
                                         ptr(self.queues), ptr(tab[4]), ptr(uni), None, C, 1, n, 0, n, A, 0, self.mode,
                                         self.seed, self.W, self.CL, g0, g0 - (ks - 1), g0, st_),
                  "decode_warp_at")
        elif self.kernel == "stream":
            check(lib.wnb_decode_stream_at(ptr(xs), ptr(aux), None, None, ptr(w["wf"]), ptr(w["bf"]), ptr(self.wstream),
                                           ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]), self.dil, self.L,
                                           ptr(self.queues), ptr(tab[4]), ptr(uni), None, C, 1, n, 0, n, self.Q, A,
                                           self.Ap, self.R, self.S, ks, 0, self.mode, self.seed, g0, g0 - (ks - 1), g0,
                                           st_),
                  "decode_stream_at")
        else:
            check(lib.wnb_decode_bf16_at(ptr(xs), ptr(aux), None, None, ptr(w["wf"]), ptr(w["bf"]), ptr(self.wstream),
                                         self.dil, self.L, ptr(self.queues), ptr(tab[4]), ptr(uni), None, C, 1, n, 0, n,
                                         self.Q, A, self.Ap, self.R, self.S, ks, 0, self.mode, self.seed, g0,
                                         g0 - (ks - 1), g0, st_),
                  "decode_bf16_at")
        self._tail = xs[:, n:].contiguous()
        # frames before each stream's next sample are no longer needed
        for slot, st, f0, f1 in spans:
            if st.sid in call.finished:
                del self._h[st.sid]
            else:
                buf = self._h[st.sid]
                f = st.aux_column(st.done) // Uc
                buf[0], buf[1] = buf[0][:, f - buf[1]:], f
        return call, xs[:, ks:]


class WaveNet(nn.Module):
    """CONDITIONAL WAVENET (reference wavenet.py:157-549).

    Args:
        n_quantize (int): Number of quantization.
        n_aux (int): Number of aux feature dimension.
        n_resch (int): Number of filter channels for residual block.
        n_skipch (int): Number of filter channels for skip connection.
        dilation_depth (int): Number of dilation depth (e.g. if set 10, max dilation = 2^(10-1)).
        dilation_repeat (int): Number of dilation repeat.
        kernel_size (int): Filter size of dilated causal convolution.
        upsampling_factor (int): Upsampling factor.
    """

    def __init__(self, n_quantize=256, n_aux=28, n_resch=512, n_skipch=256,
                 dilation_depth=10, dilation_repeat=3, kernel_size=2, upsampling_factor=0):
        super(WaveNet, self).__init__()
        self.n_aux = n_aux
        self.n_quantize = n_quantize
        self.n_resch = n_resch
        self.n_skipch = n_skipch
        self.kernel_size = kernel_size
        self.dilation_depth = dilation_depth
        self.dilation_repeat = dilation_repeat
        self.upsampling_factor = upsampling_factor

        self.dilations = [2 ** i for i in range(self.dilation_depth)] * self.dilation_repeat
        self.receptive_field = (self.kernel_size - 1) * sum(self.dilations) + 1

        # contraction precision of training (forward and backward). "fp32" = FFMA parity path, "tf32" = wgmma
        # tensor-core path, "bf16" = wgmma with both operands of every product rounded to bf16 on the per-block
        # composed path (bf16_supported(); the deferred-skip stack is tf32 only). Storage, accumulation, gradients
        # and optimizer state stay fp32 in every mode. Decode (fast_generate / batch_fast_generate) is always fp32,
        # whatever math_mode says, so that argmax decoding keeps its parity with the reference.
        self.math_mode = "fp32"
        # decode precision, separate from math_mode: "fp32" (default; argmax parity with the reference) or "bf16", the
        # opt-in tensor-core decoder of the recipe sizes (decode_bf16_supported(); any other shape raises, no fallback)
        self.decode_math = "fp32"

        # for preprocessing
        self.onehot = OneHot(self.n_quantize)
        self.causal = CausalConv1d(self.n_quantize, self.n_resch, self.kernel_size)
        if self.upsampling_factor > 0:
            self.upsampling = UpSampling(self.upsampling_factor)

        # for residual blocks
        self.dil_sigmoid = nn.ModuleList()
        self.dil_tanh = nn.ModuleList()
        self.aux_1x1_sigmoid = nn.ModuleList()
        self.aux_1x1_tanh = nn.ModuleList()
        self.skip_1x1 = nn.ModuleList()
        self.res_1x1 = nn.ModuleList()
        for d in self.dilations:
            self.dil_sigmoid += [CausalConv1d(self.n_resch, self.n_resch, self.kernel_size, d)]
            self.dil_tanh += [CausalConv1d(self.n_resch, self.n_resch, self.kernel_size, d)]
            self.aux_1x1_sigmoid += [nn.Conv1d(self.n_aux, self.n_resch, 1)]
            self.aux_1x1_tanh += [nn.Conv1d(self.n_aux, self.n_resch, 1)]
            self.skip_1x1 += [nn.Conv1d(self.n_resch, self.n_skipch, 1)]
            self.res_1x1 += [nn.Conv1d(self.n_resch, self.n_resch, 1)]

        # for postprocessing
        self.conv_post_1 = nn.Conv1d(self.n_skipch, self.n_skipch, 1)
        self.conv_post_2 = nn.Conv1d(self.n_skipch, self.n_quantize, 1)

    # -------------------------------------------------------------------------------------
    # weight packing (include/wnb200.h "Packed weight layouts"); differentiable torch ops so the
    # gradients of the packed matrices flow back to the reference-shaped parameters
    # -------------------------------------------------------------------------------------
    @property
    def n_aux_pad(self):
        return _round_up(self.n_aux, 32)

    def _math(self):
        if self.math_mode == "fp32":
            return MATH_FP32
        if self.math_mode == "tf32":
            return MATH_TF32
        if self.math_mode == "bf16":
            return MATH_BF16
        raise ValueError("math_mode should be fp32, tf32 or bf16, got %r" % (self.math_mode,))

    def _pack(self):
        R, A, Ap, ks = self.n_resch, self.n_aux, self.n_aux_pad, self.kernel_size
        L = len(self.dilations)
        st = torch.stack
        wd = torch.cat([st([m.conv.weight for m in self.dil_sigmoid]),
                        st([m.conv.weight for m in self.dil_tanh])], 1)            # (L, 2R, R, ks)
        wd = wd.permute(0, 1, 3, 2).reshape(L, 2 * R, ks * R)                       # [o][j*R + c]
        wa = torch.cat([st([m.weight for m in self.aux_1x1_sigmoid])[..., 0],
                        st([m.weight for m in self.aux_1x1_tanh])[..., 0]], 1)      # (L, 2R, A)
        wa = F.pad(wa, (0, Ap - A))
        W1 = torch.cat([wd, wa], 2).contiguous()                                    # (L, 2R, K1)
        b1 = torch.cat([st([m.conv.bias for m in self.dil_sigmoid]) + st([m.bias for m in self.aux_1x1_sigmoid]),
                        st([m.conv.bias for m in self.dil_tanh]) + st([m.bias for m in self.aux_1x1_tanh])],
                       1).contiguous()                                              # (L, 2R)
        # the last block's residual output is discarded (reference wavenet.py:230-238): its res_1x1
        # gets no gradient there, so keep it out of the graph here as well
        res_w = [m.weight if l + 1 < L else m.weight.detach() for l, m in enumerate(self.res_1x1)]
        res_b = [m.bias if l + 1 < L else m.bias.detach() for l, m in enumerate(self.res_1x1)]
        W2 = torch.cat([st(res_w)[..., 0], st([m.weight for m in self.skip_1x1])[..., 0]], 1).contiguous()
        b2 = torch.cat([st(res_b), st([m.bias for m in self.skip_1x1])], 1).contiguous()
        wf = self.causal.conv.weight.permute(2, 1, 0).contiguous()                  # (ks, Q, R)
        bf = self.causal.conv.bias
        Wp1 = self.conv_post_1.weight[..., 0].contiguous()
        Wp2 = self.conv_post_2.weight[..., 0].contiguous()
        return wf, bf, W1, b1, W2, b2, Wp1, self.conv_post_1.bias, Wp2, self.conv_post_2.bias

    def _pack_stack(self, packed):
        """Operands of the deferred-skip stack (csrc/stack.cu) from ``_pack()``'s: W2 / b2 split into the residual part
        ``W2res (L,R,R)``, ``b2res (L,R)`` and the skip GEMM operand over the concatenated gate outputs
        ``Wskip (S, L*R)`` with ``Wskip[s][l*R + c] = skip_1x1[l].weight[s][c]``, ``bskip (S) = sum_l skip_1x1[l].bias``."""
        wf, bf, W1, b1, W2, b2, Wp1, bp1, Wp2, bp2 = packed
        R, S, L = self.n_resch, self.n_skipch, len(self.dilations)
        W2res, b2res = W2[:, :R].contiguous(), b2[:, :R].contiguous()
        Wskip = W2[:, R:].permute(1, 0, 2).reshape(S, L * R).contiguous()
        bskip = b2[:, R:].sum(0)
        return wf, bf, W1, b1, W2res, b2res, Wskip, bskip, Wp1, bp1, Wp2, bp2

    def _aux(self, h, upsample=True):
        """(B, A, T or T/U) -> channels-last (B, T, Ap) with the up-sampling layer applied."""
        if h.size(1) != self.n_aux:
            raise ValueError("aux feature has %d dims, expected %d" % (h.size(1), self.n_aux))
        if self.upsampling_factor > 0 and upsample:
            return _UpsampleFn.apply(h, self.upsampling.conv.weight, self.upsampling.conv.bias, self.n_aux_pad)
        return _UpsampleFn.apply(h, None, None, self.n_aux_pad)

    def _stack_plan(self, device):
        """Copy tables + packed buffers of the one-launch weight packing (nets/packing.py); None when the deferred-skip
        stack does not cover this model."""
        if not getattr(self, "deferred_skip", True) or self.math_mode != "tf32":
            return None
        if not _lib.load().wnb_stack_supported(self.n_resch, self.n_skipch, self.n_aux_pad, self.kernel_size,
                                               len(self.dilations), MATH_TF32):
            return None
        plan = self.__dict__.get("_wnb_plan")
        if plan is None or plan.device != device or plan.stale():
            from .packing import StackPlan
            plan = StackPlan(self, device)
            self.__dict__["_wnb_plan"] = plan
        return plan

    def forward_loss(self, x, h, t, start=None):
        """Training entry of this build: mean cross entropy of ``forward(x, h)[:, start:]`` against ``t[:, start:]``
        (reference bin/train.py:533-536 with ``start = receptive_field``) as ONE autograd node -- the post network's
        logits never make a round trip through a separate loss kernel's gradient multiply.  Same value and gradients as
        ``cross_entropy(self(x, h), t, start)``."""
        start = self.receptive_field if start is None else int(start)
        if not x.is_cuda:
            raise _lib.WnbError("WaveNet.forward_loss needs CUDA tensors: this build has no CPU fallback")
        plan = self._stack_plan(x.device)
        if plan is None:
            return cross_entropy(self._forward_impl(x, h), t, start)
        return _StackTrainFn.apply(self, plan, x, h, t, start, *plan.autograd_params())

    def score(self, x, h, t, lengths, start=None, out=None):
        """Teacher-forced negative log-likelihood of held-out utterances (DESIGN.md section 6, row e1).

        ``x`` (B, T) int64 input codes, ``h`` the aux features of ``forward``, ``t`` (B, T) int64 next-sample targets
        (``utils.scoring.utterance_arrays`` aligns them as the training batches are), ``lengths`` (B,) the number of
        valid positions of each row (an int64 CUDA tensor, or a host sequence).  Scores positions ``start <= p <
        lengths[b]``; ``start`` defaults to ``receptive_field``, the training loss's start, after which no position sees
        the causal zero padding.

        Runs the forward of the model's ``math_mode`` under ``no_grad`` (two ping-ponged activation buffers; under
        fp32 and bf16 the weights are first packed with torch ops, as ``forward`` packs them), then one
        ``wnb_cross_entropy_rows`` launch.  Returns ``(nll_sum float64 (B,), count int64 (B,))`` on the device, without
        synchronising: the summed NLL in nats and the number of scored positions of each row (0, and nll 0, for a row
        with no scored position).  A row's result is bit-identical whatever else is in the batch and however far it is
        padded.  ``out`` = (nll, count): add into these instead of fresh zeroed tensors (a chain of window calls,
        ``utils.scoring.score_windows``)."""
        start = self.receptive_field if start is None else int(start)
        if not x.is_cuda:
            raise _lib.WnbError("WaveNet.score needs CUDA tensors: this build has no CPU fallback")
        lib = _lib.load()
        B, T = x.shape
        dev = x.device
        if not torch.is_tensor(lengths):
            lengths = torch.tensor([int(v) for v in lengths], dtype=torch.int64).to(dev)
        t = t.contiguous()
        if (t.dtype != torch.int64 or tuple(t.shape) != (B, T) or t.device != dev or lengths.dtype != torch.int64
                or tuple(lengths.shape) != (B,) or lengths.device != dev):
            raise ValueError("score: t should be an int64 (B, T) = %s tensor and lengths an int64 (B,) tensor on %s"
                             % ((B, T), dev))
        if start < 0:
            raise ValueError("score: start should be >= 0, got %d" % start)
        st = stream()
        if out is None:
            nll = torch.empty(B, device=dev, dtype=torch.float64)
            count = torch.empty(B, device=dev, dtype=torch.int64)
            check(lib.wnb_zero(ptr(nll), 8 * B, st), "zero")
            check(lib.wnb_zero(ptr(count), 8 * B, st), "zero")
        else:
            nll, count = out
            if (nll.dtype != torch.float64 or count.dtype != torch.int64 or tuple(nll.shape) != (B,)
                    or tuple(count.shape) != (B,) or nll.device != dev or count.device != dev):
                raise ValueError("score: out should be a float64 and an int64 (B,) = (%d,) tensor on %s" % (B, dev))
        with torch.no_grad():
            logits = self._forward_impl(x, h)
            check(lib.wnb_cross_entropy_rows(ptr(logits), ptr(t), ptr(lengths), start, ptr(nll), ptr(count), B, T,
                                             self.n_quantize, st), "cross_entropy_rows")
        return nll, count

    def _forward_impl(self, x, h, upsample=True):
        if not x.is_cuda:
            raise _lib.WnbError("WaveNet.forward needs CUDA tensors: this build has no CPU fallback")
        if upsample and PROFILE_EVENTS is None:
            plan = self._stack_plan(x.device)
            if plan is not None:
                return _StackTrainFn.apply(self, plan, x, h, None, 0, *plan.autograd_params())
        haux = self._aux(h, upsample)
        if haux.size(1) != x.size(1):
            raise ValueError("aux length %d does not match waveform length %d" % (haux.size(1), x.size(1)))
        packed = self._pack()
        meta = (self.n_quantize, self.n_resch, self.n_skipch, self.n_aux_pad, self.kernel_size,
                tuple(self.dilations), self._math())
        if getattr(self, "deferred_skip", True) and _lib.load().wnb_stack_supported(self.n_resch, self.n_skipch, self.n_aux_pad, self.kernel_size,
                                           len(self.dilations), self._math()):
            return _WaveNetStackFn.apply(x, haux, *self._pack_stack(packed), meta)
        return _WaveNetFn.apply(x, haux, *packed, meta)

    def forward(self, x, h):
        """FORWARD CALCULATION (reference wavenet.py:212-241).

        Args:
            x (Tensor): Long tensor variable with the shape (B, T).
            h (Tensor): Float tensor variable with the shape (B, n_aux, T)
                (or (B, n_aux, T / upsampling_factor) with the upsampling layer).

        Returns:
            Tensor: Float tensor variable with the shape (B, T, n_quantize).
        """
        return self._forward_impl(x, h)

    # -------------------------------------------------------------------------------------
    # generation
    # -------------------------------------------------------------------------------------
    def generate(self, x, h, n_samples, intervals=None, mode="sampling"):
        """GENERATE WAVEFORM WITH NAIVE CALCULATION (reference wavenet.py:243-307).

        O(receptive_field) work per sample through the training forward kernels; kept, like in the
        reference, as the ground truth the fast algorithm is tested against."""
        if mode not in ("sampling", "argmax"):
            logging.error("mode should be sampling or argmax")
            sys.exit(1)
        with torch.no_grad():
            if self.upsampling_factor > 0:
                h = self.upsampling(h)
            n_pad = self.receptive_field - x.size(1)
            if n_pad > 0:
                x = F.pad(x, (n_pad, 0), "constant", self.n_quantize // 2)
                h = F.pad(h, (n_pad, 0), "replicate")
            samples = x[0].tolist()
            start = time.time()
            for i in range(n_samples):
                current_idx = len(samples)
                xx = torch.tensor(samples[-self.receptive_field:], device=h.device).long().view(1, -1)
                h_ = h[:, :, current_idx - self.receptive_field: current_idx].contiguous()
                output = self._forward_impl(xx, h_, upsample=False)[0]
                if mode == "sampling":
                    posterior = F.softmax(output[-1], dim=0)
                    sample = int(torch.distributions.Categorical(posterior).sample())
                else:
                    sample = int(output[-1].argmax())
                samples.append(sample)
                if intervals is not None and (i + 1) % intervals == 0:
                    logging.info("%d/%d estimated time = %.3f sec (%.3f sec / sample)" % (
                        i + 1, n_samples,
                        (n_samples - i - 1) * ((time.time() - start) / intervals),
                        (time.time() - start) / intervals))
                    start = time.time()
        return np.array(samples[-n_samples:])

    def _decode_pack(self):
        def pad4(t):  # pad the output (last) dim of a K-major matrix to a multiple of 4
            o = t.size(-1)
            return F.pad(t, (0, _round_up(o, 4) - o)).contiguous()
        with torch.no_grad():
            wf, bf, W1, b1, W2, b2, Wp1, bp1, Wp2, bp2 = [t.detach().float() for t in self._pack()]
            R = self.n_resch
            return dict(wf=wf.contiguous(), bf=bf.contiguous(), w1d=pad4(W1.transpose(1, 2)), b1=b1,
                        w2d=pad4(W2.transpose(1, 2)), b2=b2, wp1d=pad4(Wp1.t()), bp1=bp1.contiguous(),
                        wp2d=pad4(Wp2.t()), bp2=bp2.contiguous(),
                        w2d_res=pad4(W2[:, :R].transpose(1, 2)), w2d_skip=pad4(W2[:, R:].transpose(1, 2)))

    def _decode_stream_pack(self, w):
        """One contiguous fp32 stream in consumption order (include/wnb200.h, wnb_decode_stream_at)."""
        R = self.n_resch
        parts = []
        for l in range(len(self.dilations)):
            parts += [w["w1d"][l].reshape(-1), w["w2d_res"][l].reshape(-1), w["w2d_skip"][l].reshape(-1)]
        parts += [w["wp1d"].reshape(-1), w["wp2d"].reshape(-1)]
        return torch.cat(parts).contiguous()

    def _decode_warp_pack(self, W, CL=1):
        """Warp-tile ordered stream for wnb_decode_warp_at with W (virtual) consumer warps (layout: csrc/decode_warp.cu).
        CL = 2: one stream per CTA of the cluster, back to back -- CTA r gets the tiles of warps r*W/2 .. (r+1)*W/2 - 1
        (= gate / residual channels, skip / post columns of its half) and the full bias vectors."""
        with torch.no_grad():
            wf, bf, W1, b1, W2, b2, Wp1, bp1, Wp2, bp2 = [t.detach().float() for t in self._pack()]
            L = W1.size(0)
            CH = 64 // W                     # gate / residual channels per warp
            WP = W // CL
            # W1 (L,128,160)[o][k] -> [j][w][g][lane][4]: k = 32j+lane; a lane's 2*CH values (index 4g+e) are
            # (sigmoid rows CH*w.., tanh rows CH*w..); consecutive lanes are 16 B apart (conflict-free LDS.128)
            t1 = W1.reshape(L, 2, W, CH, 5, 32).permute(0, 4, 2, 1, 3, 5)          # [L][j][w][br][cc][lane]
            t1 = t1.reshape(L, 5, W, 2 * CH // 4, 4, 32).permute(0, 1, 2, 3, 5, 4)  # [L][j][w][g][lane][4]
            # W2 res rows (L,64,64)[o][k] -> [j][w][g][lane][4]: k = 32j+lane, o = CH*w + 4g + e
            tr = W2[:, :64, :].reshape(L, W, CH, 2, 32).permute(0, 3, 1, 2, 4)     # [L][j][w][cc][lane]
            tr = tr.reshape(L, 2, W, CH // 4, 4, 32).permute(0, 1, 2, 3, 5, 4)      # [L][j][w][g][lane][4]
            # W2 skip rows (L,512,64)[o][k] -> [k][512]
            ts = W2[:, 64:, :].transpose(1, 2)                                      # [L][64 k][512]
            p1, p2 = Wp1.t(), Wp2.t()                                              # [512 k][512], [512 k][256]
            S, Q = p1.size(1), p2.size(1)
            parts = []
            for r in range(CL):
                ws = slice(r * WP, (r + 1) * WP)
                # biases ride in the stream right behind their matrices: [W1 | b1 | W2res | b2 | W2skip] per layer,
                # then [bp1 | bp2 | Wp1^T | Wp2^T]
                per_layer = torch.cat([t1[:, :, ws].reshape(L, -1), b1, tr[:, :, ws].reshape(L, -1), b2,
                                       ts[:, :, r * S // CL:(r + 1) * S // CL].reshape(L, -1)], 1).reshape(-1)
                parts += [per_layer, bp1, bp2, p1[:, r * S // CL:(r + 1) * S // CL].reshape(-1),
                          p2[:, r * Q // CL:(r + 1) * Q // CL].reshape(-1)]
            return torch.cat(parts).contiguous()

    def _decode_bf16_pack(self):
        """Per-CTA bf16 streams of the bf16 decoder, back to back, as one int16 tensor on the module's device (layout:
        csrc/decode_bf16.cu, wnb_decode_bf16_weights).  Weights are rounded to nearest even; biases stay fp32 (two 16-bit
        elements each)."""
        with torch.no_grad():
            wf, bf, W1, b1, W2, b2, Wp1, bp1, Wp2, bp2 = [t.detach().float() for t in self._pack()]
            L = W1.size(0)
            R, S, Q, ks, Ap = self.n_resch, self.n_skipch, self.n_quantize, self.kernel_size, self.n_aux_pad
            Ak = _round_up(Ap, 64)
            CR, CS, QC = R // 8, S // 8, Q // 8

            def bf(t):
                return t.to(torch.bfloat16).view(torch.int16)

            def f32(t):
                return t.contiguous().view(torch.int16)

            # W1 columns [taps j = 0..ks-2 | x(t) | aux Ap] -> [aux Ak | taps | x(t)]
            W1k = torch.cat([F.pad(W1[:, :, ks * R:], (0, Ak - Ap)), W1[:, :, :ks * R]], 2)
            parts = []
            for r in range(8):
                rows = torch.cat([torch.arange(r * CR, (r + 1) * CR), R + torch.arange(r * CR, (r + 1) * CR)])
                rrows = torch.cat([torch.arange(r * CR, (r + 1) * CR), R + torch.arange(r * CS, (r + 1) * CS)])
                rows, rrows = rows.to(W1.device), rrows.to(W1.device)
                per_layer = torch.cat([bf(_bf16_swizzle(W1k[:, rows])).reshape(L, -1), f32(b1[:, rows]).reshape(L, -1),
                                       bf(_bf16_swizzle(W2[:, rrows])).reshape(L, -1), f32(b2[:, rrows]).reshape(L, -1)], 1)
                parts += [per_layer.reshape(-1),
                          bf(_bf16_swizzle(Wp1[r * CS:(r + 1) * CS])).reshape(-1), f32(bp1[r * CS:(r + 1) * CS]),
                          bf(_bf16_swizzle(Wp2[r * QC:(r + 1) * QC])).reshape(-1), f32(bp2[r * QC:(r + 1) * QC])]
            return torch.cat(parts).contiguous()

    def _decode(self, x, h, n_samples_list, mode, uniforms=None, return_logits=False, seed=None, kernel="auto"):
        """Decode every sample at once: one call of a ``DecodeSession`` given all the aux frames, i.e. one launch over
        positions 0 .. P - 1 + max_n - 1 (after the parallel warm-up on ``warp``, ``stream`` and ``bf16``).  Returns the (B, max_n)
        int32 codes, and the (B, max_n, Q) teacher-check logits with ``return_logits``; ``last_decode_kernel`` names the
        decoder that ran.  ``x`` may be on the CPU, ``h`` may not."""
        if not h.is_cuda:
            raise _lib.WnbError("generation needs CUDA tensors: this build has no CPU fallback")
        n_list = [int(n) for n in n_samples_list]
        max_n, T0, Th = max(n_list), x.size(1), h.size(2)
        if Th * max(self.upsampling_factor, 1) < max_n + T0 - 1:
            raise ValueError("aux features too short: %d frames for %d samples" % (Th, max_n + T0))
        if max_n < 1:
            raise _lib.WnbError("decode: every requested length is 0")
        with torch.no_grad():
            s = DecodeSession(self, x.to(h.device), n_list, mode, seed, uniforms, return_logits, kernel)
            out = s.step(h)
        self.last_decode_kernel = s.kernel
        return out

    def fast_generate(self, x, h, n_samples, intervals=None, mode="sampling"):
        """GENERATE WAVEFORM WITH FAST ALGORITHM (reference wavenet.py:309-395).

        One persistent kernel launch; ``intervals`` only controls the summary log line.  Decoding is fp32 whatever
        ``math_mode`` is (argmax parity with the reference), unless ``decode_math`` is "bf16"."""
        start = time.time()
        gen = self._decode(x[:1], h[:1], [n_samples], mode)
        out = gen[0, :n_samples].cpu().numpy().astype(np.int64)
        if intervals is not None:
            el = time.time() - start
            logging.info("%d/%d generated in %.3f sec (%.6f sec / sample)" % (n_samples, n_samples, el,
                                                                              el / max(n_samples, 1)))
        return out

    def batch_fast_generate_pcm16(self, x, h, n_samples_list, intervals=None, mode="sampling"):
        """``batch_fast_generate`` + ``decode_mu_law`` + PCM_16 quantisation (reference bin/decode.py:316-319) without
        leaving the device in between: one decode launch, one gather kernel for the whole batch, 2 bytes per sample over
        PCIe.  Returns int16 arrays in COMPLETION order like ``batch_fast_generate``."""
        n_list = [int(n) for n in n_samples_list]
        pcm = codes_to_pcm16(self._decode(x, h, n_list, mode), self.n_quantize).cpu().numpy()
        order = sorted(range(len(n_list)), key=lambda b: (n_list[b], b))
        return [pcm[b, :n_list[b]].copy() for b in order]

    def batch_fast_generate(self, x, h, n_samples_list, intervals=None, mode="sampling"):
        """GENERATE WAVEFORM WITH FAST ALGORITHM IN BATCH MODE (reference wavenet.py:397-511).

        Returns the utterances in COMPLETION order (ascending length, ties by batch index) exactly
        like the reference's retirement loop (:487-509).  The caller's list is not mutated.  Decoding is fp32 whatever
        ``math_mode`` is (argmax parity with the reference), unless ``decode_math`` is "bf16"."""
        start = time.time()
        n_list = [int(n) for n in n_samples_list]
        gen = self._decode(x, h, n_list, mode).cpu().numpy().astype(np.int64)
        order = sorted(range(len(n_list)), key=lambda b: (n_list[b], b))
        outs = [gen[b, :n_list[b]].copy() for b in order]
        if intervals is not None:
            el = time.time() - start
            logging.info("%d utterances, %d samples generated in %.3f sec (%.6f sec / sample step)" % (
                len(n_list), sum(n_list), el, el / max(max(n_list), 1)))
        return outs

    def decode_session(self, x, n_samples_list=None, mode="sampling", seed=None):
        """Start a resumable decode of the batch with seed samples ``x`` (B, T0) on the GPU: feed aux frames with
        ``DecodeSession.step`` as they arrive and get the new samples back after each call.  Chunked decoding equals
        ``batch_fast_generate`` (same ``seed``, or the same ``torch.manual_seed``) bit for bit, whatever the chunk sizes.
        ``n_samples_list`` gives each utterance's length; None leaves the lengths open, so that every call decodes all the
        aux it has been given (up to the session's position limit).  The session snapshots the weights and
        ``decode_math`` now; later changes to the model do not reach it."""
        if n_samples_list is None:
            P = max(x.size(1), self.receptive_field)
            n_samples_list = [MAX_DECODE_POSITION - (P - 1)] * x.size(0)
        with torch.no_grad():
            return DecodeSession(self, x, n_samples_list, mode, seed)

    def decode_pool(self, capacity=64, mode="sampling", seed=None, park_below=None, kernel="auto"):
        """Start a continuous-batching decode pool of ``capacity`` rows, on the bf16 decoder under ``decode_math="bf16"``
        and on the fp32 warp decoder under "fp32" (the 64 res / 512 skip, ks 2 shape; another shape raises
        ``WnbError``): ``admit`` streams at any time, ``feed`` their aux frames and ``step`` to decode; a stream takes a
        free row as soon as its first frames arrive and leaves it when it finishes or is cancelled.  Stream k of a pool
        with ``seed`` S decodes what row k of a one-shot decode with seed S decodes, bit for bit: on the bf16 decoder,
        and on the warp decoder for a one-shot batch of the pool's warp form (``DecodePool``).  The pool runs in lock
        step, unless ``park_below=m`` lets it park a stream that cannot run min(m, samples left) samples until its frames
        arrive.  The pool snapshots the weights now; ``seed`` is drawn from torch's generator when not given.
        ``kernel``: "auto" (the decoder of ``decode_math``), "warp", "bf16", or "stream" for an fp32 pool on the
        streaming decoder (any shape it covers; bit-identical to one-shot ``kernel="stream"`` decoding)."""
        with torch.no_grad():
            return DecodePool(self, capacity, mode, seed, park_below, kernel)
