#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""Generate the golden vectors under tests/golden/ from the LIVE reference.

Needs a checkout of the original PytorchWaveNetVocoder (v0.1.1); the tests only read the stored vectors:

    python tests/golden/make_golden.py /path/to/PytorchWaveNetVocoder

It imports ``wavenet_vocoder.nets`` from that checkout (never copied into this repo), loads
seeded synthetic parameters (``oracle.wavenet_oracle.make_params``; numpy RandomState, so the
same arrays are rebuilt bit-for-bit by the tests on any machine) into the reference modules and
records their outputs: mu-law tables, forward logits, CE loss, every parameter gradient, and
the generate / fast_generate / batch_fast_generate index sequences.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
if len(sys.argv) != 2:
    sys.exit(__doc__)
sys.path.insert(0, os.path.abspath(sys.argv[1]))

from oracle import wavenet_oracle as O  # noqa: E402
from tests.golden.cases import FORWARD_CASES, GEN_CASES, make_inputs, make_gen_inputs, mulaw_inputs, mulaw_pcm16_domain  # noqa: E402
from wavenet_vocoder.nets import WaveNet, decode_mu_law, encode_mu_law  # noqa: E402

torch.set_num_threads(8)


def ref_model(cfg, params):
    net = WaveNet(*cfg.as_tuple())
    sd = {k: torch.from_numpy(v.copy()) for k, v in params.items()}
    net.load_state_dict(sd)
    return net


def main():
    out = {}
    # ---- mu-law ----
    x32, x64, codes = mulaw_inputs()
    out["mulaw_enc_f32"] = encode_mu_law(x32, 256)
    out["mulaw_enc_f64"] = encode_mu_law(x64, 256)
    out["mulaw_dec"] = decode_mu_law(codes, 256)
    out["mulaw_enc_pcm16"] = encode_mu_law(mulaw_pcm16_domain(), 256).astype(np.uint8)
    np.savez_compressed(os.path.join(HERE, "mulaw.npz"), **out)
    print("mulaw ok", out["mulaw_enc_f32"][:12], out["mulaw_dec"][:3])
    if "--only-mulaw" in sys.argv:
        return

    # ---- forward / loss / grads ----
    for name, (cfg_t, seed, B, T, start) in FORWARD_CASES.items():
        cfg = O.Config(*cfg_t)
        params = O.make_params(cfg, seed)
        x, h, t = make_inputs(cfg, seed, B, T)
        net = ref_model(cfg, params)
        net.train()
        y = net(torch.from_numpy(x), torch.from_numpy(h))
        loss = torch.nn.CrossEntropyLoss()(
            y[:, start:].contiguous().view(-1, cfg.n_quantize),
            torch.from_numpy(t)[:, start:].contiguous().view(-1))
        loss.backward()
        rec = {"logits": y.detach().numpy(), "loss": np.float64(loss.item())}
        for k, v in net.named_parameters():
            if v.grad is None:   # last layer's res_1x1: its output is discarded (wavenet.py:230-238)
                rec["nograd." + k] = np.zeros(1)
            else:
                rec["grad." + k] = v.grad.numpy()
        np.savez_compressed(os.path.join(HERE, "forward_%s.npz" % name), **rec)
        print("forward", name, y.shape, float(loss))

    # ---- generation (argmax, deterministic) ----
    for name, (cfg_t, seed, B, T0, n_list, naive) in GEN_CASES.items():
        cfg = O.Config(*cfg_t)
        params = O.make_params(cfg, seed)
        x, h = make_gen_inputs(cfg, seed, B, T0, n_list)
        net = ref_model(cfg, params)
        net.eval()
        rec = {}
        U = max(cfg.upsampling_factor, 1)
        with torch.no_grad():
            for b in range(B):
                n = n_list[b]
                nf = (n + T0 + U - 1) // U if cfg.upsampling_factor > 0 else n + T0
                hb = torch.from_numpy(h[b:b + 1, :, :nf])
                xb = torch.from_numpy(x[b:b + 1])
                rec["fast_%d" % b] = net.fast_generate(xb, hb, n, mode="argmax")
                if naive:
                    rec["naive_%d" % b] = net.generate(xb, hb, n, mode="argmax")
                    assert np.array_equal(rec["naive_%d" % b], rec["fast_%d" % b]), name
            if B > 1:
                outs = net.batch_fast_generate(torch.from_numpy(x), torch.from_numpy(h),
                                               list(n_list), mode="argmax")
                for i, o in enumerate(outs):
                    rec["batch_%d" % i] = o
        np.savez_compressed(os.path.join(HERE, "gen_%s.npz" % name), **rec)
        print("gen", name, {k: v.shape for k, v in rec.items()})


if __name__ == "__main__":
    main()
