# -*- coding: utf-8 -*-
"""CPU oracle for the WaveNet hot paths -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A from-scratch numpy restatement of the arithmetic in the reference's
``wavenet_vocoder/nets/wavenet.py`` (kan-bayashi/PytorchWaveNetVocoder v0.1.1) for the two
hot paths named in BASELINE.json: training forward/backward through the residual stack and
the fast-generate autoregressive loop.  Every function cites the reference file:line it
follows.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs may import this package; the product path
(``pytorchwavenetvocoder_b200``) never does and fails loudly without its CUDA library.

Parity pinning: the reference ships no golden vectors (its tests are unseeded
self-consistency checks, SURVEY.md section 4), so this oracle is pinned against the reference
module itself, imported from a checkout of the original project by
``tests/golden/make_golden.py``; the resulting vectors are committed under ``tests/golden/``
and ``tests/test_oracle_golden.py`` checks the oracle against them on every CPU run.

Parameters are a plain ``dict`` keyed by the reference's ``state_dict`` names
(``causal.conv.weight`` ...), values numpy arrays in the reference's shapes.
"""
from __future__ import division

import numpy as np


# --------------------------------------------------------------------------------------
# mu-law codec
# --------------------------------------------------------------------------------------
def encode_mu_law(x, mu=256):
    """wavenet.py:17-30.  dtype follows numpy promotion of the input (float32 stays float32
    for sign/log/abs; the division by the python-float ``np.log(1 + mu)`` keeps float32 under
    numpy>=2 for float32 arrays)."""
    mu = mu - 1
    fx = np.sign(x) * np.log(1 + mu * np.abs(x)) / np.log(1 + mu)
    return np.floor((fx + 1) / 2 * mu + 0.5).astype(np.int64)


def decode_mu_law(y, mu=256):
    """wavenet.py:33-47 (note the -0.5: not the exact inverse of encode)."""
    mu = mu - 1
    fx = (y - 0.5) / mu * 2 - 1
    x = np.sign(fx) / mu * ((1 + mu) ** np.abs(fx) - 1)
    return x


# --------------------------------------------------------------------------------------
# config helpers
# --------------------------------------------------------------------------------------
class Config(object):
    """Mirror of the WaveNet ctor arguments, wavenet.py:172-185."""

    def __init__(self, n_quantize=256, n_aux=28, n_resch=512, n_skipch=256,
                 dilation_depth=10, dilation_repeat=3, kernel_size=2, upsampling_factor=0):
        self.n_quantize = n_quantize
        self.n_aux = n_aux
        self.n_resch = n_resch
        self.n_skipch = n_skipch
        self.dilation_depth = dilation_depth
        self.dilation_repeat = dilation_repeat
        self.kernel_size = kernel_size
        self.upsampling_factor = upsampling_factor
        self.dilations = [2 ** i for i in range(dilation_depth)] * dilation_repeat  # :184
        self.receptive_field = (kernel_size - 1) * sum(self.dilations) + 1  # :185

    def as_tuple(self):
        return (self.n_quantize, self.n_aux, self.n_resch, self.n_skipch, self.dilation_depth,
                self.dilation_repeat, self.kernel_size, self.upsampling_factor)


def param_shapes(cfg):
    """state_dict key -> shape, as dumped from the live reference (wavenet.py:188-210)."""
    Q, A, R, S, ks, U = (cfg.n_quantize, cfg.n_aux, cfg.n_resch, cfg.n_skipch,
                         cfg.kernel_size, cfg.upsampling_factor)
    shapes = [("causal.conv.weight", (R, Q, ks)), ("causal.conv.bias", (R,))]
    if U > 0:
        shapes += [("upsampling.conv.weight", (1, 1, 1, U)), ("upsampling.conv.bias", (1,))]
    L = len(cfg.dilations)
    for name, shp in (("dil_sigmoid.%d.conv", (R, R, ks)), ("dil_tanh.%d.conv", (R, R, ks)),
                      ("aux_1x1_sigmoid.%d", (R, A, 1)), ("aux_1x1_tanh.%d", (R, A, 1)),
                      ("skip_1x1.%d", (S, R, 1)), ("res_1x1.%d", (R, R, 1))):
        for l in range(L):
            shapes += [((name % l) + ".weight", shp), ((name % l) + ".bias", (shp[0],))]
    shapes += [("conv_post_1.weight", (S, S, 1)), ("conv_post_1.bias", (S,)),
               ("conv_post_2.weight", (Q, S, 1)), ("conv_post_2.bias", (Q,))]
    return shapes


def make_params(cfg, seed, dtype=np.float32):
    """Seeded synthetic parameters (numpy legacy RandomState: stable across machines).

    Xavier-uniform-like conv weights as in ``initialize`` (wavenet.py:50-63) but with
    *non-zero* biases and a *non-constant* upsampling weight, because the reference's
    initialiser zeros/ones them and would hide bias/upsampling bugs (SURVEY.md 8c item 2).
    """
    rng = np.random.RandomState(seed)
    p = {}
    for name, shp in param_shapes(cfg):
        if name.startswith("upsampling"):
            if name.endswith("weight"):
                v = 1.0 + 0.2 * rng.standard_normal(shp)
            else:
                v = 0.1 * rng.standard_normal(shp)
        elif name.endswith("weight"):
            fan_out, fan_in = shp[0] * shp[2], shp[1] * shp[2]
            a = np.sqrt(6.0 / (fan_in + fan_out))
            v = rng.uniform(-a, a, size=shp)
        else:
            v = 0.05 * rng.standard_normal(shp)
        p[name] = np.ascontiguousarray(v.astype(dtype))
    return p


# --------------------------------------------------------------------------------------
# forward building blocks (all (B, C, T) like the reference)
# --------------------------------------------------------------------------------------
def causal_conv(x, W, b, d=1):
    """CausalConv1d, wavenet.py:95-121: y[t] = b + sum_k W[:,:,k] x[t-(ks-1-k)d], zero for t<0."""
    B, C, T = x.shape
    O, _, ks = W.shape
    y = np.zeros((B, O, T), dtype=x.dtype) + b[None, :, None]
    for k in range(ks):
        s = (ks - 1 - k) * d
        if s < T:
            y[:, :, s:] += np.matmul(W[:, :, k], x[:, :, :T - s])   # (O,C) @ (B,C,T') -> (B,O,T'), BLAS
    return y


def conv1x1(x, W, b):
    """nn.Conv1d(C, O, 1), wavenet.py:203-210."""
    return np.matmul(W[:, :, 0], x) + b[None, :, None]


def front_embed(x, W, b):
    """OneHot + causal conv (wavenet.py:78-92, 513-516) restated as an embedding gather:
    out[:, t] = b + sum_k W[:, x[t-(ks-1-k)] % Q, k], missing history contributes zero."""
    B, T = x.shape
    R, Q, ks = W.shape
    x = x % Q  # :88
    y = np.zeros((B, R, T), dtype=W.dtype) + b[None, :, None]
    for k in range(ks):
        s = ks - 1 - k
        if s < T:
            y[:, :, s:] += np.transpose(W[:, :, k].T[x[:, :T - s]], (0, 2, 1))
    return y


def upsample(h, w, b):
    """UpSampling, wavenet.py:124-154: ConvTranspose2d(1,1,(1,U),stride (1,U)):
    out[b,c,tU+j] = h[b,c,t] * w[j] + bias."""
    U = w.shape[-1]
    wj = w.reshape(U)
    out = h[:, :, :, None] * wj[None, None, None, :] + b.reshape(())
    return out.reshape(h.shape[0], h.shape[1], h.shape[2] * U)


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def residual_block(x, h, p, l, d):
    """_residual_forward, wavenet.py:525-536.  Returns (out, skip, cache)."""
    a = causal_conv(x, p["dil_sigmoid.%d.conv.weight" % l], p["dil_sigmoid.%d.conv.bias" % l], d) + \
        conv1x1(h, p["aux_1x1_sigmoid.%d.weight" % l], p["aux_1x1_sigmoid.%d.bias" % l])
    g = causal_conv(x, p["dil_tanh.%d.conv.weight" % l], p["dil_tanh.%d.conv.bias" % l], d) + \
        conv1x1(h, p["aux_1x1_tanh.%d.weight" % l], p["aux_1x1_tanh.%d.bias" % l])
    sg, th = sigmoid(a), np.tanh(g)
    z = sg * th
    skip = conv1x1(z, p["skip_1x1.%d.weight" % l], p["skip_1x1.%d.bias" % l])
    out = conv1x1(z, p["res_1x1.%d.weight" % l], p["res_1x1.%d.bias" % l]) + x
    return out, skip, (sg, th, z)


def postprocess(s, p):
    """_postprocess, wavenet.py:518-523; returns (B, T, Q)."""
    r0 = np.maximum(s, 0)
    h1 = conv1x1(r0, p["conv_post_1.weight"], p["conv_post_1.bias"])
    r1 = np.maximum(h1, 0)
    y = conv1x1(r1, p["conv_post_2.weight"], p["conv_post_2.bias"])
    return np.transpose(y, (0, 2, 1)), (r0, h1, r1)


def forward(cfg, p, x, h, return_cache=False):
    """WaveNet.forward, wavenet.py:212-241: x (B,T) int, h (B,A,T or T/U) -> logits (B,T,Q)."""
    out = front_embed(x, p["causal.conv.weight"], p["causal.conv.bias"])
    h_in = h
    if cfg.upsampling_factor > 0:
        h = upsample(h, p["upsampling.conv.weight"], p["upsampling.conv.bias"])
    xs, caches = [], []
    skip_sum = 0  # python 0 + left-to-right sum, wavenet.py:238
    for l, d in enumerate(cfg.dilations):
        xs.append(out)
        out, skip, c = residual_block(out, h, p, l, d)
        caches.append(c)
        skip_sum = skip_sum + skip
    y, pc = postprocess(skip_sum, p)
    if return_cache:
        return y, dict(xs=xs, caches=caches, skip_sum=skip_sum, post=pc, h=h, h_in=h_in, x=x)
    return y


def cross_entropy(logits, target, start):
    """nn.CrossEntropyLoss (mean) on [:, start:], bin/train.py:534-536.
    Returns (loss, dlogits) with dlogits zero before ``start``."""
    B, T, Q = logits.shape
    lg = logits[:, start:].reshape(-1, Q).astype(np.float64)
    tg = target[:, start:].reshape(-1)
    m = lg.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(lg - m).sum(axis=1))
    n = lg.shape[0]
    loss = float((lse - lg[np.arange(n), tg]).mean())
    sm = np.exp(lg - lse[:, None])
    sm[np.arange(n), tg] -= 1.0
    d = np.zeros((B, T, Q), dtype=logits.dtype)
    d[:, start:] = (sm / n).reshape(B, T - start, Q).astype(logits.dtype)
    return loss, d


# --------------------------------------------------------------------------------------
# manual backward (what autograd does for bin/train.py:537-538); returns grads by key
# --------------------------------------------------------------------------------------
def _conv1x1_bwd(x, W, dy):
    dW = np.matmul(dy, np.transpose(x, (0, 2, 1))).sum(axis=0)[:, :, None]   # sum_b dy[b] x[b]^T
    db = dy.sum(axis=(0, 2))
    dx = np.matmul(W[:, :, 0].T, dy)
    return dx, dW, db


def _causal_conv_bwd(x, W, dy, d):
    B, C, T = x.shape
    O, _, ks = W.shape
    dW = np.zeros_like(W)
    dx = np.zeros_like(x)
    for k in range(ks):
        s = (ks - 1 - k) * d
        if s < T:
            dW[:, :, k] = np.matmul(dy[:, :, s:], np.transpose(x[:, :, :T - s], (0, 2, 1))).sum(axis=0)
            dx[:, :, :T - s] += np.matmul(W[:, :, k].T, dy[:, :, s:])
    return dx, dW, dy.sum(axis=(0, 2))


def backward(cfg, p, cache, dlogits, relu_masks=None):
    """Gradients of every parameter given d(loss)/d(logits) (B,T,Q).

    ``relu_masks`` (test aid): {"h1": bool (B,S,T), "skip": bool (B,S,T)} replaces the two ReLU sign patterns of the
    post network (wavenet.py:518-523) by the ones another forward produced, so that a reduced-precision run can be
    compared on its arithmetic alone (a pre-activation within rounding distance of zero flips its mask, and every
    flipped element passes / blocks its whole gradient: chaotic, not an arithmetic error of the backward)."""
    g = {}
    r0, h1, r1 = cache["post"]
    dy = np.transpose(dlogits, (0, 2, 1))
    dr1, g["conv_post_2.weight"], g["conv_post_2.bias"] = _conv1x1_bwd(r1, p["conv_post_2.weight"], dy)
    dh1 = dr1 * ((h1 > 0) if relu_masks is None else relu_masks["h1"])
    dr0, g["conv_post_1.weight"], g["conv_post_1.bias"] = _conv1x1_bwd(r0, p["conv_post_1.weight"], dh1)
    dskip = dr0 * ((cache["skip_sum"] > 0) if relu_masks is None else relu_masks["skip"])
    h = cache["h"]
    dh = np.zeros_like(h)
    dout = np.zeros_like(cache["xs"][0])
    for l in reversed(range(len(cfg.dilations))):
        d = cfg.dilations[l]
        x = cache["xs"][l]
        sg, th, z = cache["caches"][l]
        dz_r, g["res_1x1.%d.weight" % l], g["res_1x1.%d.bias" % l] = \
            _conv1x1_bwd(z, p["res_1x1.%d.weight" % l], dout)
        dz_s, g["skip_1x1.%d.weight" % l], g["skip_1x1.%d.bias" % l] = \
            _conv1x1_bwd(z, p["skip_1x1.%d.weight" % l], dskip)
        dz = dz_r + dz_s
        da = dz * th * sg * (1 - sg)
        dg = dz * sg * (1 - th * th)
        dx_a, g["dil_sigmoid.%d.conv.weight" % l], g["dil_sigmoid.%d.conv.bias" % l] = \
            _causal_conv_bwd(x, p["dil_sigmoid.%d.conv.weight" % l], da, d)
        dx_g, g["dil_tanh.%d.conv.weight" % l], g["dil_tanh.%d.conv.bias" % l] = \
            _causal_conv_bwd(x, p["dil_tanh.%d.conv.weight" % l], dg, d)
        dh_a, g["aux_1x1_sigmoid.%d.weight" % l], g["aux_1x1_sigmoid.%d.bias" % l] = \
            _conv1x1_bwd(h, p["aux_1x1_sigmoid.%d.weight" % l], da)
        dh_g, g["aux_1x1_tanh.%d.weight" % l], g["aux_1x1_tanh.%d.bias" % l] = \
            _conv1x1_bwd(h, p["aux_1x1_tanh.%d.weight" % l], dg)
        dh += dh_a + dh_g
        dout = dout + dx_a + dx_g
    # front conv: scatter-add over the one-hot index
    W = p["causal.conv.weight"]
    R, Q, ks = W.shape
    x = cache["x"] % Q
    B, T = x.shape
    dW = np.zeros_like(W)
    for k in range(ks):
        s = ks - 1 - k
        if s < T:
            idx = x[:, :T - s].reshape(-1)
            contrib = np.transpose(dout[:, :, s:], (0, 2, 1)).reshape(-1, R)
            tmp = np.zeros((Q, R), dtype=W.dtype)
            np.add.at(tmp, idx, contrib)
            dW[:, :, k] = tmp.T
    g["causal.conv.weight"] = dW
    g["causal.conv.bias"] = dout.sum(axis=(0, 2))
    if cfg.upsampling_factor > 0:
        U = cfg.upsampling_factor
        h_in = cache["h_in"]
        dhr = dh.reshape(dh.shape[0], dh.shape[1], h_in.shape[2], U)
        g["upsampling.conv.weight"] = np.einsum("bctj,bct->j", dhr, h_in).reshape(1, 1, 1, U)
        g["upsampling.conv.bias"] = dh.sum().reshape(1)
    return g


# --------------------------------------------------------------------------------------
# autoregressive generation
# --------------------------------------------------------------------------------------
def _pad_inputs(cfg, p, x, h):
    """Shared prologue of generate/fast_generate, wavenet.py:257-265 / 326-334 / 416-424."""
    if cfg.upsampling_factor > 0:
        h = upsample(h, p["upsampling.conv.weight"], p["upsampling.conv.bias"])
    n_pad = cfg.receptive_field - x.shape[1]
    if n_pad > 0:
        x = np.concatenate([np.full((x.shape[0], n_pad), cfg.n_quantize // 2, dtype=x.dtype), x], axis=1)
        h = np.concatenate([np.repeat(h[:, :, :1], n_pad, axis=2), h], axis=2)
    return x, h


def _pick(logits_row, mode, u):
    if mode == "argmax":
        return int(np.argmax(logits_row))  # first max on ties, like torch CPU argmax
    if mode == "sampling":
        # inverse-CDF categorical draw from softmax(logits) with the supplied uniform u
        # (the reference uses torch.distributions.Categorical, wavenet.py:377-379, whose RNG
        #  stream cannot be reproduced outside torch; distribution is what is pinned)
        # A target below the total lands on a class whose cumulative sum rises past it, so of nonzero probability; a
        # target at or past the total (u >= 1) takes the last class of nonzero probability, like the kernels.
        m = logits_row.max()
        e = np.exp((logits_row - m).astype(np.float32))
        c = np.cumsum(e, dtype=np.float32)
        k = int(np.searchsorted(c, np.float32(u) * c[-1], side="right"))
        if k >= logits_row.shape[0]:
            k = int(np.nonzero(e > 0)[0][-1])
        return k
    raise ValueError("mode should be sampling or argmax")


def generate_naive(cfg, p, x, h, n_samples, mode="argmax", uniforms=None):
    """WaveNet.generate, wavenet.py:243-307: full network on the last rf samples per step."""
    x, h = _pad_inputs(cfg, p, x, h)
    samples = list(x[0])
    rf = cfg.receptive_field
    for i in range(n_samples):
        cur = len(samples)
        xx = np.asarray(samples[-rf:], dtype=np.int64)[None]
        hh = h[:1, :, cur - rf:cur]
        c2 = Config(*cfg.as_tuple()[:7] + (0,))
        y = forward(c2, p, xx, hh)[0]
        samples.append(_pick(y[-1], mode, None if uniforms is None else uniforms[i]))
    return np.asarray(samples[-n_samples:], dtype=np.int64)


class FifoState(object):
    """Per-layer dilation queues as ring buffers holding each layer's INPUT history
    (equivalent to the reference's output_buffer cat/slice, wavenet.py:337-350, 366-367)."""

    def __init__(self, cfg, B, dtype):
        self.q = [np.zeros((B, cfg.n_resch, (cfg.kernel_size - 1) * d), dtype=dtype)
                  for d in cfg.dilations]
        self.pos = 0


def fifo_step(cfg, p, st, x_prev, x_cur, h_col, want_logits=True):
    """One time step of the fast-generate recurrence (wavenet.py:355-375, 538-549) for a batch.

    x_prev: list of the ks-1 previous sample indices per row (arrays (B,), -1 = no history),
    x_cur (B,) current input sample, h_col (B, A) aux at this position.
    Returns logits (B,Q) (or None) and advances the queues."""
    W, b = p["causal.conv.weight"], p["causal.conv.bias"]
    R, Q, ks = W.shape
    B = x_cur.shape[0]
    cur = np.zeros((B, R), dtype=W.dtype) + b[None]
    taps = list(x_prev) + [x_cur]
    for k in range(ks):
        idx = taps[k]
        valid = idx >= 0
        cur[valid] += W[:, :, k].T[idx[valid] % Q]
    skip_sum = 0
    t = st.pos
    for l, d in enumerate(cfg.dilations):
        q = st.q[l]
        qlen = q.shape[2]
        Ws, Wt = p["dil_sigmoid.%d.conv.weight" % l], p["dil_tanh.%d.conv.weight" % l]
        a = np.zeros((B, R), dtype=cur.dtype) + p["dil_sigmoid.%d.conv.bias" % l][None]
        g = np.zeros((B, R), dtype=cur.dtype) + p["dil_tanh.%d.conv.bias" % l][None]
        for k in range(ks):
            s = (ks - 1 - k) * d
            if s == 0:
                xin = cur
            else:
                # input of this layer at time t-s; ring slot (t - s) mod qlen, zero if t-s < 0
                xin = q[:, :, (t - s) % qlen] if t - s >= 0 else np.zeros_like(cur)
            a = a + xin.dot(Ws[:, :, k].T)
            g = g + xin.dot(Wt[:, :, k].T)
        a = a + h_col.dot(p["aux_1x1_sigmoid.%d.weight" % l][:, :, 0].T) + p["aux_1x1_sigmoid.%d.bias" % l][None]
        g = g + h_col.dot(p["aux_1x1_tanh.%d.weight" % l][:, :, 0].T) + p["aux_1x1_tanh.%d.bias" % l][None]
        z = sigmoid(a) * np.tanh(g)
        if want_logits:
            skip = z.dot(p["skip_1x1.%d.weight" % l][:, :, 0].T) + p["skip_1x1.%d.bias" % l][None]
            skip_sum = skip_sum + skip
        nxt = z.dot(p["res_1x1.%d.weight" % l][:, :, 0].T) + p["res_1x1.%d.bias" % l][None] + cur
        q[:, :, t % qlen] = cur
        cur = nxt
    st.pos += 1
    if not want_logits:
        return None
    r0 = np.maximum(skip_sum, 0)
    h1 = np.maximum(r0.dot(p["conv_post_1.weight"][:, :, 0].T) + p["conv_post_1.bias"][None], 0)
    return h1.dot(p["conv_post_2.weight"][:, :, 0].T) + p["conv_post_2.bias"][None]


def batch_fast_generate(cfg, p, x, h, n_samples_list, mode="argmax", uniforms=None,
                        return_logits=False):
    """batch_fast_generate / fast_generate (wavenet.py:309-395, 397-511) restated with FIFOs.

    The reference's warm-up (full zero-padded conv over the padded prefix, :337-350) equals
    stepping the FIFOs from an all-zero state through the padded prefix positions 0..P-2
    (SURVEY.md section 7, verified there against the live reference and re-verified by
    tests/golden).  Returns a list of int64 arrays in COMPLETION order (ascending length,
    ties by original index, wavenet.py:487-509); the caller's list is not mutated."""
    n_list = list(n_samples_list)
    x, h = _pad_inputs(cfg, p, x, h)
    B, P = x.shape
    ks = cfg.kernel_size
    dtype = p["causal.conv.weight"].dtype
    st = FifoState(cfg, B, dtype)
    seq = [x[:, i].astype(np.int64) for i in range(P)]
    none = -np.ones(B, dtype=np.int64)

    def prev(pos):
        return [seq[pos - (ks - 1 - k)] if pos - (ks - 1 - k) >= 0 else none for k in range(ks - 1)]

    for pos in range(P - 1):
        fifo_step(cfg, p, st, prev(pos), seq[pos], h[:, :, pos].astype(dtype), want_logits=False)
    max_n = max(n_list)
    all_logits = []
    for i in range(max_n):
        pos = P - 1 + i
        lg = fifo_step(cfg, p, st, prev(pos), seq[pos], h[:, :, pos].astype(dtype))
        if return_logits:
            all_logits.append(lg)
        nxt = np.array([_pick(lg[b], mode, None if uniforms is None else uniforms[b][i])
                        for b in range(B)], dtype=np.int64)
        seq.append(nxt)
    gen = np.stack(seq[P:], axis=1)  # (B, max_n)
    order = sorted(range(B), key=lambda b: (n_list[b], b))
    outs = [gen[b, :n_list[b]].copy() for b in order]
    if return_logits:
        return outs, np.stack(all_logits, axis=1)
    return outs


def fast_generate(cfg, p, x, h, n_samples, mode="argmax", uniforms=None):
    """fast_generate, wavenet.py:309-395 (B=1)."""
    u = None if uniforms is None else [uniforms]
    return batch_fast_generate(cfg, p, x, h, [n_samples], mode, u)[0]
