# -*- coding: utf-8 -*-
"""``train_generator`` (reference bin/train.py:67-312, mini-batch modes) with the per-batch work on the GPU.

The reference builds every batch on the host -- window slicing, mu-law over the whole window, StandardScaler,
transpose, stack, three ``.cuda()`` copies per batch (train.py:157-185) -- in a Python prefetch thread.  At the step
times (milliseconds) that thread is the wall.  Here

* a loader thread only READS files (wav + feature frames) into pinned staging slots;
* each utterance is copied ONCE, asynchronously on a copy stream, into device ring buffers holding the
  concatenated float32 waveform and the concatenated feature frames (the reference's ``x_buffer`` / ``h_buffer``);
* one kernel launch (``wnb_make_train_batch``, csrc/loader.cu) cuts a whole batch out of the rings: windowing with
  the reference's hop arithmetic, mu-law (bit exact), scaler, (frames, D) -> (D, frames) layout, next-sample targets.

Same batches, bit for bit, as ``bin.train.train_generator`` on the same file lists (tests/test_gpu_loader.py).
``DeviceCorpusGenerator`` yields the same batches from a corpus prepared and kept on the device (utils/corpus.py,
``wnb_make_train_batch_corpus``), with no files, threads or rings.
"""
import logging
import threading
from queue import Queue

import numpy as np
import torch

from .. import _lib
from .utils import read_hdf5, read_wav


def load_pair_frames(wavfile, featfile, feature_type, upsampling_factor, use_upsampling_layer, use_speaker_code):
    """One utterance at FRAME rate: waveform float32 (n,), features (frames, D), trimmed like the reference's
    ``validate_length`` (train.py:35-64, 119-138).  For the extend_time mode (no up-sampling layer) the features stay
    at frame rate -- the device kernel indexes them per sample -- but are float64 like ``extend_time``'s output."""
    x, _ = read_wav(wavfile, dtype=np.float32)
    h = read_hdf5(featfile, "/" + feature_type)
    U = upsampling_factor
    if not use_upsampling_layer:
        h = np.asarray(h, dtype=np.float64)
    if use_speaker_code:
        sc = read_hdf5(featfile, "/speaker_code")
        h = np.concatenate([h, np.tile(sc, [h.shape[0], 1])], axis=1)
    if use_upsampling_layer:
        if x.shape[0] > h.shape[0] * U:
            x = x[:h.shape[0] * U]
        if x.shape[0] < h.shape[0] * U:
            mod_y = h.shape[0] * U - x.shape[0]
            h = h[:-(mod_y // U + 1)]
            x = x[:h.shape[0] * U]
        assert len(x) == len(h) * U
    else:
        n = min(x.shape[0], h.shape[0] * U)      # validate_length(x, extend_time(h, U))
        x = x[:n]
        h = h[:(n + U - 1) // U]
    return np.ascontiguousarray(x, dtype=np.float32), np.ascontiguousarray(h)


def _f32_scaler_mode():
    """How the installed scikit-learn transforms a float32 array (StandardScaler.transform is what the reference's
    feat_transform calls, train.py:470): 0 = float64 arithmetic rounded to float32 after the subtraction and after the
    division (scikit-learn 0.22, the reference's pin), 2 = float32 arithmetic (scikit-learn >= 1.x casts mean_ / scale_
    to the array's dtype first).  Probed, not parsed from the version string."""
    from sklearn.preprocessing import StandardScaler
    rng = np.random.RandomState(0)
    x = rng.standard_normal((64, 4)).astype(np.float32)
    sc = StandardScaler()
    sc.mean_, sc.scale_ = rng.standard_normal(4), 0.5 + rng.rand(4)
    got = sc.transform(x)
    f64 = ((x.astype(np.float64) - sc.mean_).astype(np.float32).astype(np.float64) / sc.scale_).astype(np.float32)
    f32 = (x - sc.mean_.astype(np.float32)) / sc.scale_.astype(np.float32)
    if np.array_equal(got, f64):
        return 0
    if np.array_equal(got, f32):
        return 2
    raise _lib.WnbError("unrecognised StandardScaler float32 arithmetic: use --host_loader true")


class _PinnedSlot(object):
    """One reusable pinned staging buffer of a reader thread.  Pinned memory is allocated ONCE per slot (and again only
    when an utterance is larger than anything seen): `pin_memory()` per utterance goes through cudaHostAlloc whenever
    the host allocator has no free block, which takes the driver lock the training loop's launches need."""

    def __init__(self):
        self.x = self.h = None
        self.event = None          # H2D copies of the last use of this slot (set by the consumer)

    def fill(self, x, h):
        if self.event is not None:
            self.event.synchronize()           # the previous contents have left for the device
        n, nf = x.shape[0], h.shape[0]
        if self.x is None or self.x.numel() < n:
            self.x = torch.empty(max(n, 1) * 5 // 4, dtype=torch.float32).pin_memory()
        ht = torch.from_numpy(h)
        if self.h is None or self.h.dtype != ht.dtype or self.h.shape[0] < nf or self.h.shape[1:] != ht.shape[1:]:
            self.h = torch.empty((max(nf, 1) * 5 // 4,) + tuple(ht.shape[1:]), dtype=ht.dtype).pin_memory()
        self.x[:n].copy_(torch.from_numpy(x))
        self.h[:nf].copy_(ht)
        return self.x[:n], self.h[:nf]


class WindowPlanner(object):
    """The reference's window / batch bookkeeping (train.py:117, 160-185, 202-230) on stream positions only: cut every
    window the buffer allows after each appended utterance, B consecutive windows make a batch, and at the end of an epoch
    the windows of an incomplete batch are DROPPED (the batch lists are re-created at the top of ``while True``) while the
    sample buffers carry over."""

    def __init__(self, batch_size, hop, need):
        self.B, self.hop, self.need = batch_size, hop, need
        self.tail = self.next = 0
        self.pending, self.ready = [], []

    def append(self, n, last_of_epoch):
        self.tail += n
        while self.tail - self.next >= self.need:
            self.pending.append(self.next)
            self.next += self.hop
            if len(self.pending) == self.B:
                self.ready.append(self.pending[0])
                self.pending = []
        if last_of_epoch:
            self.pending = []

    def oldest_needed(self):
        return self.ready[0] if self.ready else (self.pending[0] if self.pending else self.next)


class DeviceTrainGenerator(object):
    """Drop-in for ``train_generator(...)`` in the mini-batch modes (``batch_length`` given): ``next()`` returns
    ``((x, h), t)`` CUDA tensors -- x, t (B, T) int64, h (B, D, T/U or T) float32."""

    def __init__(self, wav_list, feat_list, receptive_field, batch_length, batch_size=1, feature_type="world",
                 n_quantize=256, mean=None, scale=None, shuffle=True, upsampling_factor=80, use_upsampling_layer=True,
                 use_speaker_code=False, device=None, ring_windows=6, prefetch=4, readers=3):
        if batch_length is None:
            raise ValueError("DeviceTrainGenerator covers the mini-batch modes; use train_generator for utterance batches")
        self.lib = _lib.load()
        self.dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.wav_list, self.feat_list = list(wav_list), list(feat_list)
        self.feature_type, self.shuffle = feature_type, shuffle
        self.U, self.use_up, self.use_spk = upsampling_factor, use_upsampling_layer, use_speaker_code
        self.B, self.mu = batch_size, n_quantize
        U = upsampling_factor
        if use_upsampling_layer:                          # train.py:99-103, 202-205
            batch_mod = (receptive_field + batch_length) % U
            logging.warning("batch length is decreased due to upsampling (%d -> %d)" % (
                batch_length, batch_length - batch_mod))
            batch_length -= batch_mod
            self.h_bs = (receptive_field + batch_length) // U
            self.T = self.h_bs * U                        # x_bs - 1
            self.Tf = self.h_bs
            self.hop = (batch_length // U) * U            # x_ss
            self.need = (self.h_bs + 1) * U               # "while len(h_buffer) > h_bs"
        else:                                             # train.py:106-110, 160-185
            win = receptive_field + batch_length
            self.T = self.Tf = win - 1
            self.hop = batch_length
            self.need = win + 1                           # "while len(x_buffer) > win"
        self.mean = None if mean is None else torch.as_tensor(np.asarray(mean, np.float64)).to(self.dev)
        self.scale = None if scale is None else torch.as_tensor(np.asarray(scale, np.float64)).to(self.dev)
        # device rings: capacity for `ring_windows` batches worth of hops plus one window
        self.cap_s = max(int(self.T + 2 + self.hop * self.B * ring_windows), 1 << 22)
        self.cap_f = self.cap_s // U + 256
        self.wave = torch.zeros(self.cap_s, dtype=torch.float32, device=self.dev)
        self.fos = None if use_upsampling_layer else torch.zeros(self.cap_s, dtype=torch.int32, device=self.dev)
        self.feat = None                                  # allocated at the first utterance (dtype / D follow the files)
        self.head_s = self.tail_s = 0                     # absolute sample positions (ring index = pos % cap_s)
        self.plan = WindowPlanner(self.B, self.hop, self.need)
        self.tail_f = 0                                   # absolute frame position of the next appended frame
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.last_batch_event = None
        self.utts = []                                    # (start_s, n, start_f, nf) of the utterances still in the ring
        # reader threads: thread k reads utterances k, k + n, ... of the (shuffled, epoch after epoch) sequence into its own
        # queue; the consumer pops the queues round-robin, so the order is the reference's
        self.n_readers = max(1, int(readers))
        self._plan_lock = threading.Lock()
        self._order = []                                  # flattened utterance sequence planned so far (file pairs)
        self._lists = (list(self.wav_list), list(self.feat_list))
        self.queues = [Queue(prefetch) for _ in range(self.n_readers)]
        self._next_q = 0
        self.stats = {"reader_s": 0.0, "utts": 0, "wait_s": 0.0, "batches": 0}
        self.threads = [threading.Thread(target=self._reader, args=(k,), daemon=True) for k in range(self.n_readers)]
        for th in self.threads:
            th.start()

    # ------------------------------------------------------------------ reader threads: file I/O only
    def _utterance(self, pos):
        """file pair at position `pos` of the infinite sequence (reference train.py:95-98, 308-312: one permutation of the
        current lists at the start and after every epoch, drawn from the global numpy RNG)"""
        with self._plan_lock:
            while pos >= len(self._order):
                wl, fl = self._lists
                if self.shuffle:
                    idx = np.random.permutation(len(wl))
                    wl, fl = [wl[i] for i in idx], [fl[i] for i in idx]
                    self._lists = (wl, fl)
                self._order.extend((w_, f_, i_ + 1 == len(wl)) for i_, (w_, f_) in enumerate(zip(wl, fl)))
            return self._order[pos]

    def _reader(self, k):
        import time
        try:
            pos = k
            slots = [_PinnedSlot() for _ in range(self.queues[k].maxsize + 3)]   # more slots than can be in flight
            i = 0
            while True:
                w, f, last_of_epoch = self._utterance(pos)
                t0 = time.time()
                x, h = load_pair_frames(w, f, self.feature_type, self.U, self.use_up, self.use_spk)
                slot = slots[i % len(slots)]
                xp, hp = slot.fill(x, h)
                self.stats["reader_s"] += time.time() - t0
                self.stats["utts"] += 1
                self.queues[k].put((xp, hp, last_of_epoch, slot))
                pos += self.n_readers
                i += 1
        except BaseException as e:     # noqa: BLE001 -- surface reader failures in the consumer
            self.queues[k].put(e)

    def _pop(self, block=True):
        q = self.queues[self._next_q]
        if not block and q.empty():
            return None
        item = q.get()
        if isinstance(item, BaseException):
            raise item
        self._next_q = (self._next_q + 1) % self.n_readers
        return item

    # ------------------------------------------------------------------ ring appends (async H2D on the copy stream)
    def _ring_copy(self, ring, pos, cap, src):
        n = src.shape[0]
        o = pos % cap
        first = min(n, cap - o)
        ring[o:o + first].copy_(src[:first], non_blocking=True)
        if first < n:
            ring[:n - first].copy_(src[first:], non_blocking=True)

    def _append(self, xp, hp, last_of_epoch=False, slot=None):
        n, nf = xp.shape[0], hp.shape[0]
        if n == 0:
            self.plan.append(0, last_of_epoch)
            return
        self.head_s = self.plan.oldest_needed()           # oldest sample a batch not launched yet still needs
        if self.feat is None:
            self.D = hp.shape[1]
            self.feat = torch.zeros(self.cap_f, self.D, dtype=hp.dtype, device=self.dev)
            self.feat_f64 = 1 if hp.dtype == torch.float64 else _f32_scaler_mode()
        if hp.dtype != self.feat.dtype:
            hp = hp.to(self.feat.dtype).pin_memory()
        while self.utts and self.utts[0][0] + self.utts[0][1] <= self.head_s:
            self.utts.pop(0)                              # fully consumed
        head_f = self.tail_f
        if self.utts:
            s_, n_, f_, nf_ = self.utts[0]
            head_f = f_ + max(self.head_s - s_, 0) // self.U
        if self.tail_s - self.head_s + n > self.cap_s or self.tail_f - head_f + nf > self.cap_f:
            raise _lib.WnbError("utterance of %d samples / %d frames does not fit the device ring (%d / %d)"
                                % (n, nf, self.cap_s, self.cap_f))
        self.utts.append((self.tail_s, n, self.tail_f, nf))
        with torch.cuda.stream(self.copy_stream):
            if self.last_batch_event is not None:
                self.copy_stream.wait_event(self.last_batch_event)   # the overwritten region was read by earlier batches
            self._ring_copy(self.wave, self.tail_s, self.cap_s, xp)
            self._ring_copy(self.feat, self.tail_f, self.cap_f, hp)
            if self.fos is not None:
                fidx = (self.tail_f + torch.arange(n, dtype=torch.int64) // self.U).to(torch.int32).pin_memory()
                self._ring_copy(self.fos, self.tail_s, self.cap_s, fidx)
                self._keep = (xp, hp, fidx)
            else:
                self._keep = (xp, hp)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.append_event = ev
        if slot is not None:
            slot.event = ev                                # the reader may refill the slot once these copies are done
        self.tail_s += n
        self.tail_f += nf
        self.plan.append(n, last_of_epoch)

    # ------------------------------------------------------------------ one batch
    def next(self):
        B, hop = self.B, self.hop
        # the reference cuts a window whenever the buffer is long enough; B consecutive windows make a batch
        import time
        t0 = time.time()
        while not self.plan.ready:
            self._append(*self._pop())
        s0 = self.plan.ready.pop(0)
        self.stats["wait_s"] += time.time() - t0
        self.stats["batches"] += 1
        t1 = time.time()
        cur = torch.cuda.current_stream(self.dev)
        cur.wait_event(self.append_event)
        x = torch.empty(B, self.T, dtype=torch.int64, device=self.dev)
        t = torch.empty(B, self.T, dtype=torch.int64, device=self.dev)
        h = torch.empty(B, self.D, self.Tf, dtype=torch.float32, device=self.dev)
        P = _lib.ptr
        _lib.check(self.lib.wnb_make_train_batch(
            P(self.wave), P(self.feat), P(self.fos), s0, hop, self.U, self.cap_s, self.cap_f, P(self.mean),
            P(self.scale), P(x), P(t), P(h), B, self.T, self.Tf, self.D, self.feat_f64, self.mu, cur.cuda_stream),
            "make_train_batch")
        ev = torch.cuda.Event()
        ev.record(cur)
        self.last_batch_event = ev
        # read ahead: whatever the reader thread has ready goes to the device now (copy stream, behind this batch's
        # kernel), so the next batches find their utterances resident and the copies overlap the training step
        while len(self.plan.ready) < 2 and self.tail_s - self.head_s < self.cap_s // 2:
            item = self._pop(block=False)
            if item is None:
                break
            self._append(*item)
        self.stats["launch_s"] = self.stats.get("launch_s", 0.0) + time.time() - t1
        return (x, h), t

    __next__ = next

    def __iter__(self):
        return self


def corpus_table(orders, first_epoch, lengths, offsets):
    """The epoch table ``wnb_make_train_batch_corpus`` searches, for epochs ``first_epoch .. first_epoch + len(orders)
    - 1`` of the stream (``orders[i]``: the utterance indices of that epoch in stream order): (starts, corpus offsets,
    table_begin, table_end).  Epoch e starts at stream position e * (sum of lengths); empty utterances take no stream
    position and are left out, so the starts increase strictly."""
    L = int(np.sum(lengths))
    starts, offs = [], []
    for i, order in enumerate(orders):
        n = lengths[order]
        st = (first_epoch + i) * L + np.concatenate([[0], np.cumsum(n)[:-1]])
        keep = n > 0
        starts.append(st[keep])
        offs.append(offsets[order][keep])
    return (np.concatenate(starts).astype(np.int64), np.concatenate(offs).astype(np.int64), first_epoch * L,
            (first_epoch + len(orders)) * L)


def corpus_index(starts, offsets, p):
    """Corpus sample of stream positions ``p``: numpy restatement of csrc/loader.cu ``corpus_index`` (the utterance with
    the largest start <= p)."""
    k = np.searchsorted(starts, p, side="right") - 1
    return offsets[k] + (p - starts[k])


class DeviceCorpusGenerator(object):
    """Drop-in for ``DeviceTrainGenerator`` in the up-sampling mini-batch mode, fed by a ``corpus.ResidentCorpus``
    instead of files: the same ``WindowPlanner`` bookkeeping over the same per-epoch ``np.random.permutation`` draws from
    the global numpy RNG gives the same sequence of batches, each cut by one ``wnb_make_train_batch_corpus`` launch
    straight from the resident int16 waveform and float32 frames.  No threads, rings or host copies per batch: the epoch
    table (stream start and corpus offset of every utterance) is uploaded when a batch reaches past the one on the
    device, about once per epoch."""

    def __init__(self, corpus, receptive_field, batch_length, batch_size=1, n_quantize=256, mean=None, scale=None,
                 shuffle=True, device=None):
        if batch_length is None or batch_length <= 0:
            raise ValueError("DeviceCorpusGenerator covers the mini-batch mode (batch_length > 0)")
        self.lib = _lib.load()
        self.dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.corpus, self.shuffle, self.B, self.mu = corpus, shuffle, batch_size, n_quantize
        U = self.U = corpus.U
        batch_mod = (receptive_field + batch_length) % U             # train.py:99-103, 202-205
        logging.warning("batch length is decreased due to upsampling (%d -> %d)" % (
            batch_length, batch_length - batch_mod))
        batch_length -= batch_mod
        self.Tf = (receptive_field + batch_length) // U
        self.T = self.Tf * U
        self.hop = (batch_length // U) * U
        self.lengths = np.asarray(corpus.lengths, dtype=np.int64)
        self.offsets = np.asarray(corpus.offsets, dtype=np.int64)
        if self.lengths.sum() == 0:
            raise ValueError("DeviceCorpusGenerator: the corpus has no samples")
        self.D = corpus.feat.size(1)
        self.feat_f64 = _f32_scaler_mode()
        self.mean = None if mean is None else torch.as_tensor(np.asarray(mean, np.float64)).to(self.dev)
        self.scale = None if scale is None else torch.as_tensor(np.asarray(scale, np.float64)).to(self.dev)
        self.plan = WindowPlanner(self.B, self.hop, (self.Tf + 1) * U)
        self._orders = []                                # utterance indices of every epoch drawn so far
        self._order = np.arange(len(self.lengths))
        self._fed = 0                                    # utterances handed to the planner
        self.table = None
        self.table_span = (0, 0)
        self.stats = {"batches": 0, "tables": 0}

    def _epoch(self, e):
        """utterance order of epoch e (reference train.py:95-98, 308-312: a permutation of the current order per epoch)"""
        while len(self._orders) <= e:
            if self.shuffle:
                self._order = self._order[np.random.permutation(len(self._order))]
            self._orders.append(self._order)
        return self._orders[e]

    def _upload(self, s0, end):
        L = int(self.lengths.sum())
        e0, e1 = s0 // L, (end - 1) // L
        starts, offs, begin, stop = corpus_table([self._epoch(e) for e in range(e0, e1 + 1)], e0, self.lengths,
                                                 self.offsets)
        self.table = torch.from_numpy(np.stack([starts, offs])).to(self.dev)
        self.table_span = (begin, stop)
        self.stats["tables"] += 1

    def next(self):
        N = len(self.lengths)
        while not self.plan.ready:
            e, i = divmod(self._fed, N)
            self.plan.append(int(self.lengths[self._epoch(e)[i]]), i + 1 == N)
            self._fed += 1
        s0 = self.plan.ready.pop(0)
        end = s0 + (self.B - 1) * self.hop + self.T + 1
        if not (self.table_span[0] <= s0 and end <= self.table_span[1]):
            self._upload(s0, end)
        x = torch.empty(self.B, self.T, dtype=torch.int64, device=self.dev)
        t = torch.empty(self.B, self.T, dtype=torch.int64, device=self.dev)
        h = torch.empty(self.B, self.D, self.Tf, dtype=torch.float32, device=self.dev)
        P = _lib.ptr
        _lib.check(self.lib.wnb_make_train_batch_corpus(
            P(self.corpus.wave), P(self.corpus.feat), P(self.table[0]), P(self.table[1]), self.table.size(1),
            self.table_span[0], self.table_span[1], s0, self.hop, self.U, P(self.mean), P(self.scale), P(x), P(t), P(h),
            self.B, self.T, self.Tf, self.D, self.feat_f64, self.mu, torch.cuda.current_stream(self.dev).cuda_stream),
            "make_train_batch_corpus")
        self.stats["batches"] += 1
        return (x, h), t

    __next__ = next

    def __iter__(self):
        return self
