# -*- coding: utf-8 -*-
"""CPU port of the reference's op sequence on torch CPU tensors -- TEST/BENCH INFRASTRUCTURE ONLY.

``oracle/wavenet_oracle.py`` is the definitional numpy restatement used for parity.  This file
restates the SAME path with the SAME torch CPU operators the reference module issues
(``F.conv1d`` with dilation + trim, one-hot scatter, ``conv_transpose2d``, cat/slice queue updates,
reference wavenet_vocoder/nets/wavenet.py:78-154, 212-241, 309-395, 397-511, 525-549) so that its
wall-clock is representative of "the reference's own CPU implementation" on the host cores.  It is
what ``bench.py`` times for ``cpu_baseline`` and for ``--impl reference`` (kind = "port": the
repository does not carry the original Python package).  It is checked against
the numpy oracle / golden vectors in tests/test_torch_port.py.

Parameters: dict keyed by the reference state_dict names -> torch tensors (fp32).
"""
import torch
import torch.nn.functional as F


def params_to_torch(p, requires_grad=False):
    out = {}
    for k, v in p.items():
        t = torch.from_numpy(v.copy()).float()
        t.requires_grad_(requires_grad)
        out[k] = t
    return out


def _causal(x, w, b, d):
    """CausalConv1d.forward, wavenet.py:108-121"""
    pad = (w.shape[2] - 1) * d
    y = F.conv1d(x, w, b, padding=pad, dilation=d)
    return y[:, :, :-pad] if pad != 0 else y


def _onehot(x, depth):
    """OneHot.forward, wavenet.py:78-92"""
    x = (x % depth).unsqueeze(2)
    oh = x.new_zeros(x.size(0), x.size(1), depth).float()
    return oh.scatter_(2, x, 1)


def _preprocess(cfg, p, x):
    return _causal(_onehot(x, cfg.n_quantize).transpose(1, 2), p["causal.conv.weight"], p["causal.conv.bias"], 1)


def _upsample(p, h):
    """UpSampling.forward, wavenet.py:141-154"""
    w = p["upsampling.conv.weight"]
    U = w.shape[-1]
    return F.conv_transpose2d(h.unsqueeze(1), w, p["upsampling.conv.bias"], stride=(1, U)).squeeze(1)


def _residual(p, l, d, x, h, last_only=False):
    """_residual_forward / _generate_residual_forward, wavenet.py:525-549"""
    a = _causal(x, p["dil_sigmoid.%d.conv.weight" % l], p["dil_sigmoid.%d.conv.bias" % l], d)
    g = _causal(x, p["dil_tanh.%d.conv.weight" % l], p["dil_tanh.%d.conv.bias" % l], d)
    if last_only:
        a, g = a[:, :, -1:], g[:, :, -1:]
    a = a + F.conv1d(h, p["aux_1x1_sigmoid.%d.weight" % l], p["aux_1x1_sigmoid.%d.bias" % l])
    g = g + F.conv1d(h, p["aux_1x1_tanh.%d.weight" % l], p["aux_1x1_tanh.%d.bias" % l])
    z = torch.sigmoid(a) * torch.tanh(g)
    skip = F.conv1d(z, p["skip_1x1.%d.weight" % l], p["skip_1x1.%d.bias" % l])
    out = F.conv1d(z, p["res_1x1.%d.weight" % l], p["res_1x1.%d.bias" % l])
    out = out + (x[:, :, -1:] if last_only else x)
    return out, skip


def _postprocess(p, x):
    y = F.conv1d(F.relu(x), p["conv_post_1.weight"], p["conv_post_1.bias"])
    y = F.conv1d(F.relu(y), p["conv_post_2.weight"], p["conv_post_2.bias"])
    return y.transpose(1, 2)


def forward(cfg, p, x, h):
    """WaveNet.forward, wavenet.py:212-241"""
    out = _preprocess(cfg, p, x)
    if cfg.upsampling_factor > 0:
        h = _upsample(p, h)
    skips = []
    for l, d in enumerate(cfg.dilations):
        out, s = _residual(p, l, d, out, h)
        skips.append(s)
    return _postprocess(p, sum(skips))


def train_step(cfg, p, opt, x, h, t):
    """bin/train.py:533-540"""
    y = forward(cfg, p, x, h)
    rf = cfg.receptive_field
    loss = F.cross_entropy(y[:, rf:].contiguous().view(-1, cfg.n_quantize), t[:, rf:].contiguous().view(-1))
    opt.zero_grad()
    loss.backward()
    opt.step()
    return loss.item()


def batch_fast_generate(cfg, p, x, h, n_samples_list, mode="argmax"):
    """batch_fast_generate, wavenet.py:397-511 (same op sequence; equal-length batches retire together)."""
    with torch.no_grad():
        max_n = max(n_samples_list)
        if cfg.upsampling_factor > 0:
            h = _upsample(p, h)
        n_pad = cfg.receptive_field - x.size(1)
        if n_pad > 0:
            x = F.pad(x, (n_pad, 0), "constant", cfg.n_quantize // 2)
            h = F.pad(h, (n_pad, 0), "replicate")
        ks = cfg.kernel_size
        out = _preprocess(cfg, p, x)
        h_ = h[:, :, :x.size(1)]
        buf, bsz = [], []
        for l, d in enumerate(cfg.dilations):
            out, _ = _residual(p, l, d, out, h_)
            bsz.append(ks - 1 if d == 2 ** (cfg.dilation_depth - 1) else d * 2 * (ks - 1))
            buf.append(out[:, :, -bsz[l] - 1: -1])
        samples = x
        for i in range(max_n):
            out = _preprocess(cfg, p, samples[:, -ks * 2 + 1:])
            h_ = h[:, :, samples.size(-1) - 1].contiguous().unsqueeze(-1)
            nbuf, skips = [], []
            for l, d in enumerate(cfg.dilations):
                out, s = _residual(p, l, d, out, h_, last_only=True)
                out = torch.cat([buf[l], out], dim=2)
                nbuf.append(out[:, :, -bsz[l]:])
                skips.append(s)
            buf = nbuf
            y = _postprocess(p, sum(skips))[:, -1]
            if mode == "argmax":
                smp = y.argmax(-1)
            else:
                smp = torch.distributions.Categorical(F.softmax(y, dim=-1)).sample()
            samples = torch.cat([samples, smp.view(-1, 1)], dim=1)
        gen = samples[:, -max_n:].numpy()
        order = sorted(range(len(n_samples_list)), key=lambda b: (n_samples_list[b], b))
        return [gen[b, :n_samples_list[b]].copy() for b in order]
