# -*- coding: utf-8 -*-
"""Host side of ``wnb_pack_weights`` (include/wnb200.h): the copy tables that turn the reference-shaped
``nn.Parameter`` set of ``WaveNet`` (reference nets/wavenet.py:188-210) into the packed kernel operands of the
deferred-skip stack (csrc/stack.cu) -- and the packed gradients back into one flat ``.grad`` buffer -- with ONE kernel
launch per direction instead of ~100 torch cat/stack/permute/pad launches and their autograd mirror per step.

Built once per (model, device); rebuilt only when a parameter's storage moves.
"""
import numpy as np
import torch

from .. import _lib

DESC = np.dtype([("src", "<i8"), ("src2", "<i8"), ("dst", "<i8"),
                 ("n0", "<i4"), ("n1", "<i4"), ("n2", "<i4"),
                 ("ss0", "<i4"), ("ss1", "<i4"), ("ss2", "<i4"),
                 ("ds0", "<i4"), ("ds1", "<i4"), ("ds2", "<i4"),
                 ("op", "<i4"), ("flags", "<i4"), ("nsum", "<i4")])
assert DESC.itemsize == 72
COPY, ADD2, SUMPTR = 0, 1, 2
SRC_ABS = 1


def _align(n, a=64):
    return (n + a - 1) // a * a


class _Sections(object):
    """Named sections of one flat fp32 buffer (offsets in floats, each 256-byte aligned)."""

    def __init__(self):
        self.off, self.shape, self.size = {}, {}, 0

    def add(self, name, *shape):
        self.off[name] = self.size
        self.shape[name] = tuple(shape)
        self.size += _align(int(np.prod(shape)))

    def view(self, buf, name):
        n = int(np.prod(self.shape[name]))
        return buf[self.off[name]:self.off[name] + n].view(self.shape[name])


class StackPlan(object):
    """Packed-parameter / packed-gradient layouts and the two copy tables for one WaveNet on one device."""

    def __init__(self, net, device):
        R, S, Q, ks, A, Ap = net.n_resch, net.n_skipch, net.n_quantize, net.kernel_size, net.n_aux, net.n_aux_pad
        L, U = len(net.dilations), net.upsampling_factor
        K1 = ks * R + Ap
        self.dims = dict(R=R, S=S, Q=Q, ks=ks, A=A, Ap=Ap, L=L, U=U, K1=K1)
        self.device = device
        P, G = _Sections(), _Sections()
        P.add("wf", ks, Q, R); P.add("bf", R)
        P.add("W1", L, 2 * R, K1); P.add("b1", L, 2 * R)
        P.add("W2res", L, R, R); P.add("b2res", L, R)
        P.add("Wskip", S, L * R); P.add("bskip", S)
        P.add("Wp1", S, S); P.add("bp1", S); P.add("Wp2", Q, S); P.add("bp2", Q)
        P.add("w1t", L, K1, 2 * R); P.add("wgate", L, 3 * R, K1 + R); P.add("wskt", L * R, S)
        P.add("wp1t", S, S); P.add("wp2t", S, Q)
        G.add("wf", ks, Q, R); G.add("bf", R)
        G.add("W1", L, 2 * R, K1); G.add("b1", L, 2 * R)
        G.add("W2res", L, R, R); G.add("b2res", L, R)
        G.add("Wskip", S, L * R); G.add("bskip", S)
        G.add("Wp1", S, S); G.add("bp1", S); G.add("Wp2", Q, S); G.add("bp2", Q)
        G.add("upw", max(U, 1)); G.add("upb", 1)
        self.P, self.G = P, G
        # persistent packed-parameter buffer: zero blocks (aux padding, wgate's off-diagonal blocks) are written once
        self.pbuf = torch.zeros(P.size, dtype=torch.float32, device=device)
        self.params = list(net.named_parameters())
        self.ptrs = None
        self._build(net)

    # ---------------------------------------------------------------------------------------------
    def stale(self):
        """parameter storage moved since the tables were built?  Checked in full every 32nd call, on three sentinels
        otherwise (187 ``data_ptr()`` calls per training step were 0.1 ms of host time)."""
        self._calls = getattr(self, "_calls", 0) + 1
        if self._calls % 32 == 1:
            return self.ptrs != tuple(p.data_ptr() for _, p in self.params)
        ps = self.params
        return (ps[0][1].data_ptr(), ps[len(ps) // 2][1].data_ptr(), ps[-1][1].data_ptr()) != \
            (self.ptrs[0], self.ptrs[len(ps) // 2], self.ptrs[-1])

    def _build(self, net):
        d = self.dims
        R, S, Q, ks, A, L, U, K1 = d["R"], d["S"], d["Q"], d["ks"], d["A"], d["L"], d["U"], d["K1"]
        P, G = self.P, self.G
        prm = dict(self.params)
        for n_, p in self.params:
            if p.dtype != torch.float32 or not p.is_contiguous() or p.device != self.device:
                raise _lib.WnbError("parameter %s must be contiguous fp32 on %s" % (n_, self.device))
        self.ptrs = tuple(p.data_ptr() for _, p in self.params)
        ptr = lambda name: prm[name].data_ptr()  # noqa: E731
        pk = []

        def cp(src, dst, n, ss, ds, op=COPY, src2=0, nsum=0, flags=SRC_ABS):
            pk.append((src, src2, dst, n[0], n[1], n[2], ss[0], ss[1], ss[2], ds[0], ds[1], ds[2], op, flags, nsum))

        # ---- pack: parameters -> P ----
        # (transposing entries iterate in SOURCE order: a strided read stalls its thread, a strided write does not)
        cp(ptr("causal.conv.weight"), P.off["wf"], (R, Q, ks), (Q * ks, ks, 1), (1, R, Q * R))
        cp(ptr("causal.conv.bias"), P.off["bf"], (1, 1, R), (0, 0, 1), (0, 0, 1))
        Kg = K1 + R
        skip_bias_ptrs = []
        for l in range(L):
            w1 = P.off["W1"] + l * 2 * R * K1
            w1t = P.off["w1t"] + l * K1 * 2 * R
            wg = P.off["wgate"] + l * 3 * R * Kg
            for br, nm in enumerate(("sigmoid", "tanh")):
                dw = ptr("dil_%s.%d.conv.weight" % (nm, l))         # (R, R, ks)  [o][c][j]
                aw = ptr("aux_1x1_%s.%d.weight" % (nm, l))          # (R, A, 1)   [o][a]
                # W1[l][br*R + o][j*R + c]
                cp(dw, w1 + br * R * K1, (R, R, ks), (R * ks, ks, 1), (K1, 1, R))
                cp(aw, w1 + br * R * K1 + ks * R, (1, R, A), (0, A, 1), (0, K1, 1))
                # wgate[l][br*R + o][j*R + c]  (rows of pitch K1 + R)
                cp(dw, wg + br * R * Kg, (R, R, ks), (R * ks, ks, 1), (Kg, 1, R))
                cp(aw, wg + br * R * Kg + ks * R, (1, R, A), (0, A, 1), (0, Kg, 1))
                # w1t[l][j*R + c][br*R + o]
                cp(dw, w1t + br * R, (R, R, ks), (R * ks, ks, 1), (1, 2 * R, R * 2 * R))
                cp(aw, w1t + ks * R * 2 * R + br * R, (1, R, A), (0, A, 1), (0, 1, 2 * R))
                cp(ptr("dil_%s.%d.conv.bias" % (nm, l)), P.off["b1"] + l * 2 * R + br * R, (1, 1, R), (0, 0, 1), (0, 0, 1),
                   op=ADD2, src2=ptr("aux_1x1_%s.%d.bias" % (nm, l)))
            rw = ptr("res_1x1.%d.weight" % l)                        # (R, R, 1) [o][c]
            cp(rw, P.off["W2res"] + l * R * R, (1, 1, R * R), (0, 0, 1), (0, 0, 1))
            cp(ptr("res_1x1.%d.bias" % l), P.off["b2res"] + l * R, (1, 1, R), (0, 0, 1), (0, 0, 1))
            # wgate[l][2R + c][K1 + o] = W2res[l][o][c]
            cp(rw, wg + 2 * R * Kg + K1, (1, R, R), (0, R, 1), (0, 1, Kg))
            sw = ptr("skip_1x1.%d.weight" % l)                       # (S, R, 1) [s][c]
            cp(sw, P.off["Wskip"] + l * R, (1, S, R), (0, R, 1), (0, L * R, 1))
            cp(sw, P.off["wskt"] + l * R * S, (1, S, R), (0, R, 1), (0, 1, S))
            skip_bias_ptrs.append(ptr("skip_1x1.%d.bias" % l))
        self.skip_bias_table = torch.tensor(skip_bias_ptrs, dtype=torch.int64, device=self.device)
        cp(self.skip_bias_table.data_ptr(), P.off["bskip"], (1, 1, S), (0, 0, 1), (0, 0, 1), op=SUMPTR, nsum=L)
        cp(ptr("conv_post_1.weight"), P.off["Wp1"], (1, 1, S * S), (0, 0, 1), (0, 0, 1))
        cp(ptr("conv_post_1.weight"), P.off["wp1t"], (1, S, S), (0, S, 1), (0, 1, S))
        cp(ptr("conv_post_1.bias"), P.off["bp1"], (1, 1, S), (0, 0, 1), (0, 0, 1))
        cp(ptr("conv_post_2.weight"), P.off["Wp2"], (1, 1, Q * S), (0, 0, 1), (0, 0, 1))
        cp(ptr("conv_post_2.weight"), P.off["wp2t"], (1, Q, S), (0, S, 1), (0, 1, Q))
        cp(ptr("conv_post_2.bias"), P.off["bp2"], (1, 1, Q), (0, 0, 1), (0, 0, 1))
        self.pack_table = self._upload(pk)
        self.n_pack = self.pack_table.numel() // DESC.itemsize

        # ---- unpack: G -> flat gradient buffer (one 16-byte aligned slice per parameter, parameters() order) ----
        # gap-free layout: parameters whose size is a multiple of 4 floats first (parameters() order), the others (the
        # 1-element up-sampling bias) last -- every slice of the first kind is 16-byte aligned without padding, and the
        # .grad views come out of ONE torch.split call
        self.grad_off, self.grad_names = {}, []
        off = 0
        with_grad = []
        for name, p in self.params:
            if name in ("res_1x1.%d.weight" % (L - 1), "res_1x1.%d.bias" % (L - 1)):
                continue     # reference: the last block's residual output is discarded -> no gradient (wavenet.py:230-238)
            if name.startswith("upsampling") and U == 0:
                continue
            with_grad.append((name, p))
        for name, p in [t for t in with_grad if t[1].numel() % 4 == 0] + [t for t in with_grad if t[1].numel() % 4 != 0]:
            self.grad_off[name] = off
            self.grad_names.append(name)
            off += p.numel()
        self.grad_size = off
        self._split_sizes = [dict(self.params)[n].numel() for n in self.grad_names]
        self._split_shapes = [tuple(dict(self.params)[n].shape) for n in self.grad_names]
        self._param_slot = [self.grad_names.index(n) if n in self.grad_off else -1 for n, _ in self.params]
        pk = []
        go = self.grad_off

        def up(src, name, n, ss, ds):
            pk.append((src, 0, go[name], n[0], n[1], n[2], ss[0], ss[1], ss[2], ds[0], ds[1], ds[2], COPY, 0, 0))

        up(G.off["wf"], "causal.conv.weight", (ks, Q, R), (Q * R, R, 1), (1, ks, Q * ks))
        up(G.off["bf"], "causal.conv.bias", (1, 1, R), (0, 0, 1), (0, 0, 1))
        if U > 0:
            up(G.off["upw"], "upsampling.conv.weight", (1, 1, U), (0, 0, 1), (0, 0, 1))
            up(G.off["upb"], "upsampling.conv.bias", (1, 1, 1), (0, 0, 1), (0, 0, 1))
        for l in range(L):
            w1 = G.off["W1"] + l * 2 * R * K1
            for br, nm in enumerate(("sigmoid", "tanh")):
                up(w1 + br * R * K1, "dil_%s.%d.conv.weight" % (nm, l), (R, ks, R), (K1, R, 1), (R * ks, 1, ks))
                up(w1 + br * R * K1 + ks * R, "aux_1x1_%s.%d.weight" % (nm, l), (1, R, A), (0, K1, 1), (0, A, 1))
                for bn in ("dil_%s.%d.conv.bias", "aux_1x1_%s.%d.bias"):
                    up(G.off["b1"] + l * 2 * R + br * R, bn % (nm, l), (1, 1, R), (0, 0, 1), (0, 0, 1))
            if l + 1 < L:
                up(G.off["W2res"] + l * R * R, "res_1x1.%d.weight" % l, (1, 1, R * R), (0, 0, 1), (0, 0, 1))
                up(G.off["b2res"] + l * R, "res_1x1.%d.bias" % l, (1, 1, R), (0, 0, 1), (0, 0, 1))
            up(G.off["Wskip"] + l * R, "skip_1x1.%d.weight" % l, (1, S, R), (0, L * R, 1), (0, R, 1))
            up(G.off["bskip"], "skip_1x1.%d.bias" % l, (1, 1, S), (0, 0, 1), (0, 0, 1))
        up(G.off["Wp1"], "conv_post_1.weight", (1, 1, S * S), (0, 0, 1), (0, 0, 1))
        up(G.off["bp1"], "conv_post_1.bias", (1, 1, S), (0, 0, 1), (0, 0, 1))
        up(G.off["Wp2"], "conv_post_2.weight", (1, 1, Q * S), (0, 0, 1), (0, 0, 1))
        up(G.off["bp2"], "conv_post_2.bias", (1, 1, Q), (0, 0, 1), (0, 0, 1))
        self.unpack_table = self._upload(pk)
        self.n_unpack = self.unpack_table.numel() // DESC.itemsize

    @staticmethod
    def _split(rows, limit=16384):
        """Break large entries into pieces of <= `limit` elements along their outermost non-trivial dimension, so that the
        work per block row of pack_kernel is even (one 262 144-element entry otherwise sets the kernel time)."""
        out = []
        for r in rows:
            src, src2, dst, n0, n1, n2, ss0, ss1, ss2, ds0, ds1, ds2, op, flags, nsum = r
            if n0 * n1 * n2 <= limit or op == SUMPTR:
                out.append(r)
                continue
            if n0 > 1:
                step = max(1, limit // (n1 * n2))
                for a in range(0, n0, step):
                    m = min(step, n0 - a)
                    out.append((src + (a * ss0) * (4 if flags & SRC_ABS else 1), src2 + ((a * ss0) * 4 if src2 else 0),
                                dst + a * ds0, m, n1, n2, ss0, ss1, ss2, ds0, ds1, ds2, op, flags, nsum))
            else:
                if n1 > 1:
                    step = max(1, limit // n2)
                    for a in range(0, n1, step):
                        m = min(step, n1 - a)
                        out.append((src + (a * ss1) * (4 if flags & SRC_ABS else 1), src2 + ((a * ss1) * 4 if src2 else 0),
                                    dst + a * ds1, 1, m, n2, ss0, ss1, ss2, ds0, ds1, ds2, op, flags, nsum))
                else:
                    for a in range(0, n2, limit):
                        m = min(limit, n2 - a)
                        out.append((src + (a * ss2) * (4 if flags & SRC_ABS else 1), src2 + ((a * ss2) * 4 if src2 else 0),
                                    dst + a * ds2, 1, 1, m, ss0, ss1, ss2, ds0, ds1, ds2, op, flags, nsum))
        return out

    def _upload(self, rows):
        rows = self._split(rows)
        arr = np.zeros(len(rows), dtype=DESC)
        for i, r in enumerate(rows):
            arr[i] = r
        return torch.from_numpy(arr.view(np.uint8).copy()).to(self.device)

    # ---------------------------------------------------------------------------------------------
    def autograd_params(self):
        """The parameters handed to ``_StackTrainFn.apply``: the modules' own under grad mode, detached views
        otherwise.  ``Function.forward`` runs with grad mode off whatever the caller's, so it tells a no-grad call
        (ping-ponged activations, nothing saved) from a training call by ``needs_input_grad`` alone."""
        if torch.is_grad_enabled():
            return [p for _, p in self.params]
        return [p.detach() for _, p in self.params]

    def pack(self, stream):
        lib = _lib.load()
        _lib.check(lib.wnb_pack_weights(self.pack_table.data_ptr(), self.n_pack, None, self.pbuf.data_ptr(), None,
                                        stream), "pack_weights")

    def p(self, name):
        return self.P.view(self.pbuf, name)

    def unpack(self, gbuf, flat, scale, stream):
        lib = _lib.load()
        _lib.check(lib.wnb_pack_weights(self.unpack_table.data_ptr(), self.n_unpack, gbuf.data_ptr(), flat.data_ptr(),
                                        None if scale is None else scale.data_ptr(), stream), "pack_weights(unpack)")

    def grad_views(self, flat):
        """one view per parameter in ``self.params`` order (None where the reference has no gradient either)"""
        parts = flat.split(self._split_sizes)
        views = [q.view(shp) for q, shp in zip(parts, self._split_shapes)]
        return [None if k < 0 else views[k] for k in self._param_slot]
