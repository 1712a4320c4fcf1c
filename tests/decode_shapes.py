# -*- coding: utf-8 -*-
"""The shape table of tests/test_gpu_decode_shapes.py and tests/test_decode_shapes_host.py: one row per branch of the
two fp32 launch rules that the decode-form tests do not reach.

``wnb_decode_stream_supported`` (decode_stream.cu ``stream_plan``) sends a model to the streaming decoder when every
padded width fits 256 consumer lanes and a 32 KB ring chunk, L <= 64, R, S and Ap are multiples of 4 and the work area
plus two ring slots fits 227 KB; every other shape runs on the direct decoder (decode.cu), which takes any width, halves
its utterances per CTA (NU) until its carve-up fits 220 KB, and refuses L > 64 or more than 227 KB at NU 1.

Each row: ``shape`` (Q, A, R, S, depth, repeat, ks, U) as ``oracle.Config`` takes it, ``dil`` the dilations that
replace the config's (None: the config's own; depth x repeat sets the layer count either way), ``rule`` ("stream":
auto runs the streaming decoder; "direct": auto runs the direct one and ``kernel="stream"`` raises; "none": neither
covers it and decoding raises), ``batches`` (B as a function of the SM count), ``max_n`` the longest utterance, and
``reaches`` what the row is there for."""
SMS_H100 = 132

ONE = (lambda n: 3,)
ROWS = {
    # ---- the streaming rule covers these: auto = streaming decoder with its parallel warm-up; direct run by name ----
    "q1024": dict(shape=(1024, 28, 64, 64, 4, 2, 2, 4), dil=None, rule="stream", batches=ONE, max_n=24,
                  reaches="Qp 1 024: 256 lanes, parts 1; 32 classes per sampler lane"),
    "q1022": dict(shape=(1022, 28, 64, 64, 4, 2, 2, 4), dil=None, rule="stream", batches=ONE, max_n=24,
                  reaches="2 padded logit columns; the last sampler lane holds 30 classes"),
    "odd_parts": dict(shape=(33, 28, 12, 12, 4, 2, 2, 0), dil=None, rule="stream",
                      batches=(lambda n: 3, lambda n: n + 5, lambda n: 2 * n + 5), max_n=16,
                      reaches="parts 42 (O1 24) / 85 (Or, Os, Sp 12) / 28 (Qp 36): idle threads, K = 12 < parts; "
                              "Q 33: sampler lanes with 1 class and with none; NU 1 / 2 / 4, last CTA part empty"),
    "widest": dict(shape=(256, 256, 512, 1024, 4, 5, 2, 0), dil=None, rule="stream",
                   batches=(lambda n: 3, lambda n: 2 * n + 5), max_n=12,
                   reaches="O1 = Os = Sp = 1 024 (256 lanes, parts 1); at B > 2 SMs NU halves from 4 to 2"),
    "smem_edge": dict(shape=(256, 80, 512, 256, 6, 6, 3, 0), dil=[1, 2, 3, 4, 5, 6] * 6, rule="stream", batches=ONE,
                      max_n=12, reaches="512/256 ks 3 Ap 96 at L 36: the last L with two ring slots"),
    "ks1": dict(shape=(256, 28, 64, 64, 4, 1, 1, 4), dil=None, rule="stream", batches=ONE, max_n=24,
                reaches="ks 1: no queues, no taps"),
    "ks4": dict(shape=(256, 28, 64, 64, 3, 2, 4, 4), dil=[1, 3, 37, 2, 5, 6], rule="stream", batches=ONE, max_n=24,
                reaches="ks 4: taps j = 0, 1, 2; dilations 1, 3, 5, 6 and 37 > max_n; queue wrap"),
    "ks5": dict(shape=(256, 28, 64, 64, 3, 2, 5, 0), dil=[5, 1, 3, 37, 2, 1], rule="stream", batches=ONE, max_n=24,
                reaches="ks 5: taps j = 0 .. 3; dilations 1, 3, 5 and 37 > max_n; queue wrap"),
    "l64": dict(shape=(256, 28, 4, 1024, 8, 8, 2, 0), dil=None, rule="stream", batches=ONE, max_n=12,
                reaches="L = 64 (kMaxLayersS); Or 4 (1 lane, parts 256), Os = Sp = 1 024 (256 lanes)"),
    # ---- the streaming rule refuses these: auto = direct, kernel="stream" raises ----
    "d1": dict(shape=(256, 28, 6, 8, 3, 1, 2, 0), dil=None, rule="direct", batches=(lambda n: 3, lambda n: n + 5),
               max_n=24, reaches="R 6: the scalar regions end at 2 mod 4 floats at NU 1 (378), at 0 mod 4 at NU 2"),
    "odd_rs_q255": dict(shape=(255, 28, 7, 9, 5, 1, 3, 0), dil=None, rule="direct", batches=ONE, max_n=24,
                        reaches="odd R and S, Q 255: padded O1, O2, Sp and Qp; scalar regions end at 3 mod 4"),
    "r516": dict(shape=(256, 28, 516, 256, 3, 1, 2, 0), dil=None, rule="direct", batches=ONE, max_n=16,
                 reaches="R 516: O1 1 032 (258 lanes) through the wide-output loop"),
    "s1028_q1028": dict(shape=(1028, 28, 64, 1028, 3, 1, 2, 0), dil=None, rule="direct", batches=ONE, max_n=16,
                        reaches="S 1 028, Q 1 028: O2 1 092, Sp and Qp 1 028 through the wide-output loop"),
    "smem_edge_l37": dict(shape=(256, 80, 512, 256, 37, 1, 3, 0), dil=[1, 2, 3, 4, 5, 6] * 6 + [7], rule="direct",
                          batches=ONE, max_n=12, reaches="512/256 ks 3 Ap 96 at L 37: too large for two ring slots"),
    "direct_nu_halves": dict(shape=(256, 28, 254, 256, 11, 2, 3, 0), dil=[1, 2, 3] * 7 + [1], rule="direct",
                             batches=(lambda n: 2 * n + 5,), max_n=8,
                             reaches="R 254 ks 3 L 22: NU 4 needs more than 220 KB, the launcher halves it to 2"),
    # ---- neither decoder covers these ----
    "l65": dict(shape=(256, 28, 4, 4, 13, 5, 2, 0), dil=[1] * 65, rule="none", batches=ONE, max_n=4,
                reaches="65 layers: over both decoders' layer limit"),
    "smem_over": dict(shape=(30000, 28, 4, 4, 1, 1, 2, 0), dil=None, rule="none", batches=ONE, max_n=4,
                      reaches="Q 30 000: the direct carve-up needs 235 KB at NU 1"),
}


def round4(v):
    return (v + 3) & ~3


def n_aux_pad(A):
    return (A + 31) // 32 * 32


def dilations(row):
    """the row's dilations"""
    Q, A, R, S, depth, repeat, ks, U = row["shape"]
    return list(row["dil"]) if row["dil"] is not None else [2 ** i for i in range(depth)] * repeat


def kernel_dims(row):
    """(Q, Ap, R, S, ks, L) as the decoders take them"""
    Q, A, R, S, depth, repeat, ks, U = row["shape"]
    return Q, n_aux_pad(A), R, S, ks, len(dilations(row))


def direct_scalar_floats(NU, Q, Ap, R, S, ks, L):
    """decode.cu decode_scalar_floats: floats of the scalar regions xcat .. qtap of NU utterances"""
    return NU * (ks * R + Ap + 2 * R + 2 * S + round4(Q) + Ap + (ks - 1) * L * R)


def direct_partial_offset(NU, Q, Ap, R, S, ks, L):
    """decode.cu decode_partial_offset: where the float4 partial sums start, rounded up to 4 floats"""
    return round4(direct_scalar_floats(NU, Q, Ap, R, S, ks, L))


def direct_plan(Q, Ap, R, S, ks, L, NU):
    """wnb_decode_at's launch rule: (NU after halving, shared-memory bytes), or None when it refuses the shape"""
    if L > 64:
        return None
    omax = max(round4(2 * R), round4(R + S), round4(S), round4(Q), 1024)
    while True:
        smem = 4 * (direct_partial_offset(NU, Q, Ap, R, S, ks, L) + NU * omax)
        if smem <= 220 * 1024 or NU == 1:
            break
        NU //= 2
    return (NU, smem) if smem <= 227 * 1024 else None


def first_nu(B, sms):
    """utterances per CTA both decoders start from"""
    return 4 if B > 2 * sms else 2 if B > sms else 1
