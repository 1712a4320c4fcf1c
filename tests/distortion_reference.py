# -*- coding: utf-8 -*-
"""Float64 numpy restatement of csrc/distortion.cu (wnb_mcd_aligned, wnb_mcd_dtw) with the kernels' operation order:
numpy's elementwise float64 operations round each result once and never fuse, as __dsub_rn / __dmul_rn / __dadd_rn /
__dsqrt_rn do.  Shared by the CPU tier (tests/test_distortion_host.py) and the GPU tier (tests/test_gpu_distortion.py)."""
import numpy as np


def _widen(frames):
    return np.asarray(np.asarray(frames, dtype=np.float32), dtype=np.float64)


def frame_dists(a, b):
    """dist of frames a[t] and b[t] (arrays of equal shape (n, D + 1)): squares of columns 1 .. D added in ascending d."""
    a, b = _widen(a), _widen(b)
    s = np.zeros(a.shape[0])
    for d in range(1, a.shape[1]):
        e = a[:, d] - b[:, d]
        s = s + e * e
    return np.sqrt(s)


def dist_matrix(ref, dec):
    """(Tr, Td) dist of every reference frame against every decoded frame, in the order of frame_dists."""
    r, q = _widen(ref), _widen(dec)
    s = np.zeros((r.shape[0], q.shape[0]))
    for d in range(1, r.shape[1]):
        e = r[:, d][:, None] - q[:, d][None, :]
        s = s + e * e
    return np.sqrt(s)


def butterfly32(v):
    """Lane 0's value after the xor butterfly v[l] += v[l ^ o], o = 16, 8, 4, 2, 1, over each row of 32 lanes."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


def aligned(ref, dec):
    """(sum, n) of wnb_mcd_aligned: dists of frames t < n = min(Tr, Td) in 32-frame chunks (zeros past n), each chunk
    an xor butterfly, the chunk sums added in ascending order from 0.0."""
    n = min(len(ref), len(dec))
    dist = frame_dists(np.asarray(ref)[:n], np.asarray(dec)[:n])
    chunks = -(-n // 32)
    v = np.zeros(chunks * 32)
    v[:n] = dist
    acc = 0.0
    for c in butterfly32(v.reshape(chunks, 32)):
        acc = acc + c
    return float(acc), n


def dtw(ref, dec, dist=None):
    """(sum, path) of wnb_mcd_dtw: the accumulated cost swept over anti-diagonals (one vectorised step per diagonal),
    ties to (i-1, j-1), then (i-1, j), then (i, j-1); the path from (0, 0) to (Tr-1, Td-1) as an (n, 2) int array and
    sum = C(Tr-1, Td-1).  ``dist`` overrides the local distance matrix (hand-built tie cases)."""
    Dm = dist_matrix(ref, dec) if dist is None else np.asarray(dist, dtype=np.float64)
    Tr, Td = Dm.shape
    C = np.empty((Tr, Td))
    step = np.zeros((Tr, Td), dtype=np.int8)      # 0 diagonal, 1 (i-1, j), 2 (i, j-1), 3 the start
    C[0, 0] = Dm[0, 0]
    step[0, 0] = 3
    for k in range(1, Tr + Td - 1):
        i = np.arange(max(0, k - Td + 1), min(k, Tr - 1) + 1)
        j = k - i
        up = np.where(i > 0, C[np.maximum(i - 1, 0), j], np.inf)
        left = np.where(j > 0, C[i, np.maximum(j - 1, 0)], np.inf)
        diag = np.where((i > 0) & (j > 0), C[np.maximum(i - 1, 0), np.maximum(j - 1, 0)], np.inf)
        best, s = diag, np.zeros(len(i), dtype=np.int8)
        take = up < best
        best, s = np.where(take, up, best), np.where(take, 1, s)
        take = left < best
        best, s = np.where(take, left, best), np.where(take, 2, s)
        C[i, j] = Dm[i, j] + best
        step[i, j] = s
    path = [(Tr - 1, Td - 1)]
    i, j = Tr - 1, Td - 1
    while i > 0 or j > 0:
        s = step[i, j]
        if s == 0:
            i, j = i - 1, j - 1
        elif s == 1:
            i -= 1
        else:
            j -= 1
        path.append((i, j))
    return float(C[Tr - 1, Td - 1]), np.array(path[::-1], dtype=np.int64)


def dtw_brute(dist):
    """Every monotone path from (0, 0) to the last cell by exhaustive recursion, each with its cost added in forward
    order: returns (least cost, the paths that have it).  For tiny matrices."""
    Dm = np.asarray(dist, dtype=np.float64)
    Tr, Td = Dm.shape
    found = []

    def walk(i, j, acc, path):
        acc = acc + Dm[i, j]
        path = path + [(i, j)]
        if i == Tr - 1 and j == Td - 1:
            found.append((acc, path))
            return
        if i + 1 < Tr and j + 1 < Td:
            walk(i + 1, j + 1, acc, path)
        if i + 1 < Tr:
            walk(i + 1, j, acc, path)
        if j + 1 < Td:
            walk(i, j + 1, acc, path)

    walk(0, 0, 0.0, [])
    least = min(c for c, _ in found)
    return float(least), [np.array(p, dtype=np.int64) for c, p in found if c == least]


def path_sum(ref, dec, path):
    """Sum of dist along ``path`` added in forward order from 0.0 (equals C(Tr-1, Td-1) bit for bit)."""
    Dm = dist_matrix(ref, dec)
    acc = 0.0
    for i, j in path:
        acc = acc + Dm[i, j]
    return float(acc)
