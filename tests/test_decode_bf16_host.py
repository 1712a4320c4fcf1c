# -*- coding: utf-8 -*-
"""CPU tier: host logic of the bf16 decoder (csrc/decode_bf16.cu) without a GPU -- shape coverage, stream and queue
sizes, the per-CTA weight stream against a naive restatement of its documented layout -- and a ptxas check that the
kernel neither spills nor has its wgmma serialised."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from pytorchwavenetvocoder_b200 import _lib, build


def test_supported_and_sizes():
    lib = _lib.load()
    assert lib.wnb_decode_bf16_supported(256, 32, 512, 256, 2, 30) == 1      # arctic recipe
    assert lib.wnb_decode_bf16_supported(256, 96, 512, 256, 3, 10) == 1      # ljspeech recipe
    assert lib.wnb_decode_bf16_supported(256, 32, 256, 256, 2, 8) == 1
    assert lib.wnb_decode_bf16_supported(256, 32, 512, 512, 2, 30) == 1
    assert lib.wnb_decode_bf16_supported(256, 32, 64, 512, 2, 30) == 0       # BASELINE 64/512: decode_warp
    assert lib.wnb_decode_bf16_supported(256, 32, 512, 256, 4, 30) == 0      # bad kernel size
    assert lib.wnb_decode_bf16_supported(256, 32, 512, 256, 1, 30) == 0
    assert lib.wnb_decode_bf16_supported(512, 32, 512, 256, 2, 30) == 0      # Q != 256
    assert lib.wnb_decode_bf16_supported(256, 256, 512, 256, 3, 30) == 0     # aux rows + 3 stages exceed 227 KB
    assert lib.wnb_decode_bf16_supported(256, 32, 512, 256, 2, 65) == 0
    dil = (ctypes.c_int32 * 4)(1, 2, 4, 8)
    assert lib.wnb_decode_bf16_workspace(64, 512, 3, dil, 4) == 1 * 2 * 15 * 512 * 64 * 2
    assert lib.wnb_decode_bf16_workspace(65, 512, 2, dil, 4) == 2 * 15 * 512 * 64 * 2
    rc = lib.wnb_decode_bf16_at(None, None, None, None, None, None, None, dil, 4, None, None, None, None, 2, 1, 5, 0, 10,
                                256, 28, 32, 512, 256, 2, 0, 0, 0, 0, 0, 0, None)
    assert rc == -1 and b"null pointer" in lib.wnb_last_error()


def _swz(tile):
    """naive: (N, 64) tile -> (N, 64) in the 128B swizzle, element by element"""
    N = tile.shape[0]
    out = np.zeros_like(tile)
    for n in range(N):
        for k in range(64):
            out[n, ((k // 8) ^ (n % 8)) * 8 + k % 8] = tile[n, k]
    return out


def _chunks(W):
    return [_swz(W[:, c:c + 64]).reshape(-1) for c in range(0, W.shape[1], 64)]


def test_weight_stream_layout():
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(1)
    Q, A, R, S, ks = 256, 28, 64, 128, 3
    net = WaveNet(Q, A, R, S, 2, 1, ks, 0)
    for prm in net.parameters():
        torch.nn.init.normal_(prm, std=0.1)
    got = net._decode_bf16_pack().numpy()
    assert got.size == _lib.load().wnb_decode_bf16_weights(Q, 32, R, S, ks, 2)
    sd = {k: v.detach().float() for k, v in net.state_dict().items()}
    bfv = lambda t: t.to(torch.bfloat16).view(torch.int16).numpy()          # noqa: E731
    f32v = lambda t: t.contiguous().view(torch.int16).numpy()               # noqa: E731
    CR, CS, Ak = R // 8, S // 8, 64
    want = []
    for r in range(8):
        ch = list(range(r * CR, (r + 1) * CR))
        for l in range(2):
            rows = []
            for branch in ("sigmoid", "tanh"):
                wd = sd["dil_%s.%d.conv.weight" % (branch, l)]          # (R, R, ks)
                wa = sd["aux_1x1_%s.%d.weight" % (branch, l)][:, :, 0]  # (R, A)
                for c in ch:
                    aux = torch.zeros(Ak)
                    aux[:A] = wa[c]
                    rows.append(torch.cat([aux] + [wd[c, :, j] for j in range(ks)]))
            W = bfv(torch.stack(rows))
            b1 = torch.cat([sd["dil_sigmoid.%d.conv.bias" % l][ch] + sd["aux_1x1_sigmoid.%d.bias" % l][ch],
                            sd["dil_tanh.%d.conv.bias" % l][ch] + sd["aux_1x1_tanh.%d.bias" % l][ch]])
            res_rows = [sd["res_1x1.%d.weight" % l][c, :, 0] for c in ch]
            skip_rows = [sd["skip_1x1.%d.weight" % l][s, :, 0] for s in range(r * CS, (r + 1) * CS)]
            W2 = bfv(torch.stack(res_rows + skip_rows))
            b2 = torch.cat([sd["res_1x1.%d.bias" % l][ch], sd["skip_1x1.%d.bias" % l][r * CS:(r + 1) * CS]])
            want += _chunks(W) + [f32v(b1)] + _chunks(W2) + [f32v(b2)]
        want += _chunks(bfv(sd["conv_post_1.weight"][r * CS:(r + 1) * CS, :, 0])) + \
            [f32v(sd["conv_post_1.bias"][r * CS:(r + 1) * CS])]
        want += _chunks(bfv(sd["conv_post_2.weight"][32 * r:32 * (r + 1), :, 0])) + \
            [f32v(sd["conv_post_2.bias"][32 * r:32 * (r + 1)])]
    assert np.array_equal(got, np.concatenate(want))


def test_kernel_compiles_without_spills_or_serialised_wgmma():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "decode_bf16.cu"),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    assert not [line for line in text.splitlines() if "C7510" in line or "C7513" in line], text
    spills = re.findall(r"Function properties for (\S*decode_bf16_kernel\S*)\n\s*\d+ bytes stack frame, (\d+) bytes "
                        r"spill stores, (\d+) bytes spill loads", text)
    assert len(spills) == 3, text
    assert all(int(s) == 0 and int(ld) == 0 for _, s, ld in spills), spills
