# -*- coding: utf-8 -*-
"""Cost of streaming the MLSA noise-shaping restoration filter (utils/mlsa.py MlsaStreamFilter) beside decoding.

    python tools/mlsa_stream_times.py [--calls 200] [--samples 4000] [--batch 64] [--json out.json]

* filter: the time of one ``MlsaStreamFilter.filter`` call (CUDA events around ``--calls`` back-to-back calls, so the
  host work between launches counts) for 1, 8 and 64 streams with chunks of 80 and 1 600 int16 samples, order 24, pd 4;
* session: the time of one 1-frame (80-sample) chunk of a decode session (``step_pcm16``, host clock around a
  synchronise, median over the calls after the first) without and with the filter on its rows, alternating the two
  runs, on the 64/512 fp32 warp decoder and the arctic 512/256 bf16 decoder, ``--batch`` utterances.
Prints the card and its power limit, read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.decode_session_times import SHAPES, card  # noqa: E402


def coef24():
    from pytorchwavenetvocoder_b200.utils.mlsa import convert_mcep_to_mlsa_coef
    return convert_mcep_to_mlsa_coef(np.random.RandomState(0).randn(25) * 0.6, 0.5, 0.41)


def filter_ms(streams, chunk, calls):
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter
    rng = np.random.RandomState(streams * 7 + chunk)
    x = torch.from_numpy(np.int16(np.clip(np.cumsum(rng.randn(streams, chunk), axis=1) * 30, -30000, 30000))).cuda()
    filt = MlsaStreamFilter(coef24(), 0.41, 4)
    chunks = {k: x[k] for k in range(streams)}
    for _ in range(3):
        filt.filter(chunks)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        filt.filter(chunks)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def session_chunk_ms(net, x, h, n, filtered):
    """median host time of one 1-frame step_pcm16 call (around a synchronise), filter included when ``filtered``"""
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter
    s = net.decode_session(x, [n] * x.size(0), "sampling", seed=1)
    filt = MlsaStreamFilter(coef24(), 0.41, 4) if filtered else None
    times, f = [], 0
    while not s.done:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = s.step_pcm16(h[:, :, f:f + 1])
        if filt is not None:
            filt.filter({b: out[b, :c] for b, c in enumerate(s.last_counts)})
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        f += 1
    return float(np.median(times[1:])) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--samples", type=int, default=4000)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200.nets import WaveNet
    name, q = card()
    print("card: %s, power limit: %s" % (name, q))
    rows = []
    for streams in (1, 8, 64):
        for chunk in (80, 1600):
            ms = filter_ms(streams, chunk, args.calls)
            rows.append({"what": "filter", "streams": streams, "chunk_samples": chunk, "ms_per_call": ms})
            print("filter: %2d streams x %4d samples, order 24: %.3f ms per call" % (streams, chunk, ms))
    torch.manual_seed(0)
    with torch.no_grad():
        for sname, (cfg, dm) in SHAPES.items():
            net = WaveNet(*cfg).cuda().eval()
            net.decode_math = dm
            B, U, n = args.batch, cfg[-1], args.samples
            rng = np.random.RandomState(B)
            x = torch.from_numpy(rng.randint(0, 256, size=(B, 1))).cuda()
            h = torch.from_numpy(rng.standard_normal((B, cfg[1], n // U + 2)).astype(np.float32)).cuda()
            session_chunk_ms(net, x, h, 4 * U, True)        # warm: module load, packing
            res = {False: [], True: []}
            for rep in range(2):
                for filtered in (False, True):
                    res[filtered].append(session_chunk_ms(net, x, h, n, filtered))
            plain, filt = float(np.median(res[False])), float(np.median(res[True]))
            rows.append({"what": "session", "shape": sname, "B": B, "chunk_samples": U, "ms_per_chunk": plain,
                         "ms_per_chunk_filtered": filt, "runs": res[False] + res[True]})
            print("session %-22s B=%d, 1-frame chunks: %.3f ms without the filter, %.3f ms with it (+%.3f ms)"
                  % (sname, B, plain, filt, filt - plain))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit": q, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
