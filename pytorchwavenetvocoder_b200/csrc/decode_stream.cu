// decode_stream.cu -- persistent fast-generate kernel, v2: weight STREAM through a shared-memory ring.
//
// The per-sample dependency chain (front -> L gated blocks -> post -> pick) cannot be parallelised over
// time, but the weights it consumes are the same 8.6 MB, in the same order, every step.  So a dedicated
// producer warp streams them from L2 into a ring of shared-memory slots with cp.async.bulk (TMA bulk
// copy, completion on an mbarrier) continuously -- across layer and step boundaries, never waiting for
// the arithmetic -- while 8 consumer warps run the recurrence out of shared memory.  The L2 latency
// that dominated v1 (decode.cu: dependent LDGs inside every GEMV) disappears from the chain; a step
// costs max(weight stream time, smem-bound GEMV time).  Teacher-forced warm-up steps stream only the
// gate and residual matrices (2.9 MB instead of 8.6 MB).
//
// Stream layout (built by nets/wavenet.py::_decode_stream_pack), all K-major [K rows][O cols], O % 4 == 0:
//   per layer l:  W1d [K1][O1] | W2res [R][Or] | W2skip [R][Os]      then  wp1d [S][Sp] | wp2d [S][Qp]
// A chunk is a whole number of rows (<= kChunkBytes); producer and consumers derive the identical chunk
// sequence from the segment shapes, so no table is needed.
//
// Same numerics as v1: fp32 FFMA, python-order skip sum, first-max argmax, Philox inverse-CDF sampling.
#include "common.cuh"
#include "tc_ptx.cuh"

namespace wnb {

constexpr int kConsThreads = 256;
constexpr int kStreamThreads = kConsThreads + 32;  // + producer warp
constexpr int kChunkBytes = 32 * 1024;
constexpr int kMaxLayersS = 64;

struct StreamParams {
  int32_t* xs; const float* h; const float* up_w; const float* up_b;
  const float *wf, *bf, *b1, *b2, *bp1, *bp2;
  const float* stream;       // packed weights (see header comment)
  float* queues; const int32_t* n_samples; const float* uniforms; float* logits_out;
  int B, P, max_n, n_pad, Th, Q, A, Ap, R, S, ks, U, mode, L;
  int pos0, i0, i_last, h_last, stride_xs;   // the call's window (common.cuh DecodeWindow)
  int O1, Or, Os, Sp, Qp;    // padded widths
  int nslot;
  unsigned long long seed;
  long long layer_stride, off_w2res, off_w2skip, off_p1, off_p2;  // float offsets inside the stream
  int dil[kMaxLayersS];
  long long qoff[kMaxLayersS];
  long long q_per_utt;
};

__device__ __forceinline__ int rows_per_chunk(int O, int parts) {
  int r = kChunkBytes / (O * 4);
  if (r > parts) r = (r / parts) * parts;
  return r < 1 ? 1 : r;
}
__device__ __forceinline__ int parts_for(int O) {
  const int lanes = O >> 2;
  return lanes >= kConsThreads ? 1 : kConsThreads / lanes;
}

__device__ __forceinline__ void bulk_g2s(void* smem, const void* gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(ptx::smem_u32(smem)), "l"(gmem), "r"(bytes), "r"(ptx::smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void cons_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

struct Ring {
  unsigned char* base; uint64_t* full; uint64_t* empty; int nslot; uint32_t idx;
};

// ---- producer side: push one K-major matrix through the ring
__device__ __forceinline__ void produce_segment(Ring& r, const float* src, int K, int O) {
  const int rpc = rows_per_chunk(O, parts_for(O));
  for (int k0 = 0; k0 < K; k0 += rpc) {
    const int rows = min(rpc, K - k0);
    const uint32_t bytes = (uint32_t)rows * O * 4;
    const int slot = r.idx % r.nslot;
    ptx::mbar_wait(&r.empty[slot], ((r.idx / r.nslot) & 1) ^ 1);
    ptx::mbar_arrive_expect_tx(&r.full[slot], bytes);
    bulk_g2s(r.base + (size_t)slot * kChunkBytes, src + (size_t)k0 * O, bytes, &r.full[slot]);
    r.idx++;
  }
}

// ---- consumer side: partial[part][u][o] = sum_{k in part} W[k][o] * x[u][k]
template <int NU, bool RELU_X>
__device__ __forceinline__ int consume_segment(Ring& r, int K, int O, const float* __restrict__ x, int ldx,
                                               float* __restrict__ partial) {
  const int tid = threadIdx.x, lanes = O >> 2;
  const int parts = parts_for(O);
  const int rpc = rows_per_chunk(O, parts);
  const int lane = tid % lanes, part = tid / lanes;
  const bool active = part < parts && lanes <= kConsThreads;
  float4 acc0[NU], acc1[NU];
#pragma unroll
  for (int u = 0; u < NU; u++) acc0[u] = acc1[u] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k0 = 0; k0 < K; k0 += rpc) {
    const int rows = min(rpc, K - k0);
    const int slot = r.idx % r.nslot;
    ptx::mbar_wait(&r.full[slot], (r.idx / r.nslot) & 1);
    if (active) {
      const float4* w = reinterpret_cast<const float4*>(r.base + (size_t)slot * kChunkBytes) + lane;
      int rr = part;
      for (; rr + parts < rows; rr += 2 * parts) {
        const float4 w0 = w[(size_t)rr * lanes], w1 = w[(size_t)(rr + parts) * lanes];
#pragma unroll
        for (int u = 0; u < NU; u++) {
          float x0 = x[u * ldx + k0 + rr], x1 = x[u * ldx + k0 + rr + parts];
          if (RELU_X) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          acc0[u].x = fmaf(w0.x, x0, acc0[u].x); acc0[u].y = fmaf(w0.y, x0, acc0[u].y);
          acc0[u].z = fmaf(w0.z, x0, acc0[u].z); acc0[u].w = fmaf(w0.w, x0, acc0[u].w);
          acc1[u].x = fmaf(w1.x, x1, acc1[u].x); acc1[u].y = fmaf(w1.y, x1, acc1[u].y);
          acc1[u].z = fmaf(w1.z, x1, acc1[u].z); acc1[u].w = fmaf(w1.w, x1, acc1[u].w);
        }
      }
      if (rr < rows) {
        const float4 w0 = w[(size_t)rr * lanes];
#pragma unroll
        for (int u = 0; u < NU; u++) {
          float x0 = x[u * ldx + k0 + rr];
          if (RELU_X) x0 = fmaxf(x0, 0.f);
          acc0[u].x = fmaf(w0.x, x0, acc0[u].x); acc0[u].y = fmaf(w0.y, x0, acc0[u].y);
          acc0[u].z = fmaf(w0.z, x0, acc0[u].z); acc0[u].w = fmaf(w0.w, x0, acc0[u].w);
        }
      }
    }
    __syncwarp();
    if ((tid & 31) == 0) ptx::mbar_arrive(&r.empty[slot]);
    r.idx++;
  }
  if (active) {
#pragma unroll
    for (int u = 0; u < NU; u++) {
      float4 v = make_float4(acc0[u].x + acc1[u].x, acc0[u].y + acc1[u].y, acc0[u].z + acc1[u].z,
                             acc0[u].w + acc1[u].w);
      reinterpret_cast<float4*>(partial + ((size_t)part * NU + u) * O)[lane] = v;
    }
  }
  return parts;
}

__device__ __forceinline__ float reduce_parts_s(const float* partial, int parts, int NU, int O, int u, int o) {
  float s = 0.f;
  for (int p = 0; p < parts; p++) s += partial[((size_t)p * NU + u) * O + o];
  return s;
}

__device__ __forceinline__ void philox4x32_10s(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                               uint32_t k1, uint32_t (&out)[4]) {
#pragma unroll
  for (int i = 0; i < 10; i++) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

template <int NU>
__global__ void __launch_bounds__(kStreamThreads, 1) decode_stream_kernel(const StreamParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int R = p.R, S = p.S, Q = p.Q, Ap = p.Ap, ks = p.ks, L = p.L;
  const int K1 = ks * R + Ap;
  const int ntap = (ks - 1) * L;
  // carve-up: ring first (128 B aligned), then barriers, then the float work area
  unsigned char* ring_base = smem_raw;
  uint64_t* full = reinterpret_cast<uint64_t*>(ring_base + (size_t)p.nslot * kChunkBytes);
  uint64_t* empty = full + p.nslot;
  float* fw = reinterpret_cast<float*>(empty + p.nslot);
  float* xcat = fw;                            // [NU][K1]
  float* cur = xcat + NU * K1;                 // [NU][R]
  float* zs = cur + NU * R;                    // [NU][R]
  float* skipacc = zs + NU * R;                // [NU][S]
  float* h1 = skipacc + NU * S;                // [NU][S]
  float* logit = h1 + NU * S;                  // [NU][Qp]
  float* hcol = logit + NU * p.Qp;             // [NU][Ap]
  float* qtap = hcol + NU * Ap;                // [NU][ntap][R]
  float* partial = qtap + (size_t)NU * ntap * R;  // [parts][NU][O]
  __shared__ int s_n[NU];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int u0 = blockIdx.x * NU;
  const int stride_xs = p.stride_xs;

  if (tid == 0) {
    for (int i = 0; i < p.nslot; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], kConsThreads / 32);
    }
    ptx::fence_barrier_init();
  }
  if (tid < NU) s_n[tid] = (u0 + tid < p.B) ? p.i0 + p.n_samples[u0 + tid] : 0;   // absolute end
  __syncthreads();
  int nmax = 0;
#pragma unroll
  for (int u = 0; u < NU; u++) nmax = max(nmax, s_n[u]);
  if (nmax <= p.i0) return;
  const int last_pos = p.P - 1 + nmax - 1;
  Ring ring{ring_base, full, empty, p.nslot, 0u};

  if (warp == kConsThreads / 32) {
    // ================================ producer warp ================================
    if (lane == 0) {
      for (int pos = p.pos0; pos <= last_pos; pos++) {
        const bool want = pos >= p.P - 1;
        for (int l = 0; l < L; l++) {
          const float* base = p.stream + (size_t)l * p.layer_stride;
          produce_segment(ring, base, K1, p.O1);
          produce_segment(ring, base + p.off_w2res, R, p.Or);
          if (want) produce_segment(ring, base + p.off_w2skip, R, p.Os);
        }
        if (want) {
          produce_segment(ring, p.stream + p.off_p1, S, p.Sp);
          produce_segment(ring, p.stream + p.off_p2, S, p.Qp);
        }
      }
    }
    return;
  }

  // ================================ consumer warps ================================
  for (int pos = p.pos0; pos <= last_pos; pos++) {
    const bool want = pos >= p.P - 1;
    for (int e = tid; e < NU * R; e += kConsThreads) {
      const int u = e / R, r = e - u * R;
      const int ug = min(u0 + u, p.B - 1);
      float v = __ldg(p.bf + r);
      for (int k = 0; k < ks; k++) {
        const int pp = pos - (ks - 1 - k);
        if (pp >= 0) {
          int q = p.xs[(size_t)ug * stride_xs + pp] % Q;
          if (q < 0) q += Q;
          v += __ldg(p.wf + ((size_t)k * Q + q) * R + r);
        }
      }
      cur[e] = v;
    }
    for (int e = tid; e < NU * Ap; e += kConsThreads) {
      const int u = e / Ap, a = e - u * Ap;
      const int ug = min(u0 + u, p.B - 1);
      float v = 0.f;
      if (a < p.A) {
        const int j = max(pos - p.n_pad, 0);
        if (p.U > 0) {
          const int tf = min(j / p.U, p.h_last), jj = j % p.U;
          v = fmaf(__ldg(p.h + ((size_t)ug * p.A + a) * p.Th + tf), __ldg(p.up_w + jj), __ldg(p.up_b));
        } else {
          v = __ldg(p.h + ((size_t)ug * p.A + a) * p.Th + min(j, p.h_last));
        }
      }
      hcol[e] = v;
    }
    for (int e = tid; e < NU * ntap * R; e += kConsThreads) {
      const int r = e % R;
      const int tp = (e / R) % ntap;
      const int u = e / (R * ntap);
      const int ug = min(u0 + u, p.B - 1);
      const int l = tp / (ks - 1), j = tp - l * (ks - 1);
      const int d = p.dil[l];
      const int s = (ks - 1 - j) * d;
      float v = 0.f;
      if (pos - s >= 0) {
        const int qlen = (ks - 1) * d;
        const float* q = p.queues + (size_t)ug * p.q_per_utt + p.qoff[l];
        v = __ldcg(q + (size_t)((pos - s) % qlen) * R + r);
      }
      qtap[e] = v;
    }
    cons_sync();

    for (int l = 0; l < L; l++) {
      const int d = p.dil[l];
      for (int e = tid; e < NU * K1; e += kConsThreads) {
        const int u = e / K1, k = e - u * K1;
        float v;
        if (k < (ks - 1) * R) {
          const int j = k / R, r = k - j * R;
          v = qtap[((size_t)u * ntap + l * (ks - 1) + j) * R + r];
        } else if (k < ks * R) {
          v = cur[u * R + (k - (ks - 1) * R)];
        } else {
          v = hcol[u * Ap + (k - ks * R)];
        }
        xcat[e] = v;
      }
      if (ks > 1) {
        const int qlen = (ks - 1) * d;
        for (int e = tid; e < NU * R; e += kConsThreads) {
          const int u = e / R, r = e - u * R;
          if (u0 + u < p.B) {
            float* q = p.queues + (size_t)(u0 + u) * p.q_per_utt + p.qoff[l];
            __stcg(q + (size_t)(pos % qlen) * R + r, cur[e]);
          }
        }
      }
      cons_sync();
      int parts = consume_segment<NU, false>(ring, K1, p.O1, xcat, K1, partial);
      cons_sync();
      for (int e = tid; e < NU * R; e += kConsThreads) {
        const int u = e / R, c = e - u * R;
        const float a = reduce_parts_s(partial, parts, NU, p.O1, u, c) + __ldg(p.b1 + (size_t)l * 2 * R + c);
        const float g = reduce_parts_s(partial, parts, NU, p.O1, u, R + c) + __ldg(p.b1 + (size_t)l * 2 * R + R + c);
        zs[e] = sigmoidf_(a) * tanhf(g);
      }
      cons_sync();
      parts = consume_segment<NU, false>(ring, R, p.Or, zs, R, partial);
      cons_sync();
      for (int e = tid; e < NU * R; e += kConsThreads) {
        const int u = e / R, o = e - u * R;
        cur[e] += reduce_parts_s(partial, parts, NU, p.Or, u, o) + __ldg(p.b2 + (size_t)l * (R + S) + o);
      }
      if (want) {
        cons_sync();   // partial is about to be overwritten
        parts = consume_segment<NU, false>(ring, R, p.Os, zs, R, partial);
        cons_sync();
        for (int e = tid; e < NU * S; e += kConsThreads) {
          const int u = e / S, o = e - u * S;
          const float v = reduce_parts_s(partial, parts, NU, p.Os, u, o) + __ldg(p.b2 + (size_t)l * (R + S) + R + o);
          float* dst = skipacc + u * S + o;
          *dst = (l == 0) ? v : (*dst + v);  // python `0 + s0 + s1 ...`, wavenet.py:374
        }
      }
      cons_sync();
    }

    if (want) {
      int parts = consume_segment<NU, true>(ring, S, p.Sp, skipacc, S, partial);
      cons_sync();
      for (int e = tid; e < NU * S; e += kConsThreads) {
        const int u = e / S, o = e - u * S;
        h1[e] = fmaxf(reduce_parts_s(partial, parts, NU, p.Sp, u, o) + __ldg(p.bp1 + o), 0.f);
      }
      cons_sync();
      parts = consume_segment<NU, false>(ring, S, p.Qp, h1, S, partial);
      cons_sync();
      const int i = pos - (p.P - 1);
      for (int e = tid; e < NU * Q; e += kConsThreads) {
        const int u = e / Q, o = e - u * Q;
        const float v = reduce_parts_s(partial, parts, NU, p.Qp, u, o) + __ldg(p.bp2 + o);
        logit[u * p.Qp + o] = v;
        if (p.logits_out && u0 + u < p.B && i < s_n[u])
          p.logits_out[((size_t)(u0 + u) * p.max_n + i) * Q + o] = v;
      }
      cons_sync();
      if (warp < NU) {
        const int u = warp;
        const float* lg = logit + u * p.Qp;
        const int chunk = (Q + 31) / 32;
        const int q0 = lane * chunk, q1 = min(q0 + chunk, Q);
        float best = -INFINITY;
        int bi = 0x7fffffff;
        for (int q = q0; q < q1; q++)
          if (lg[q] > best) { best = lg[q]; bi = q; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        int pick = bi;
        if (p.mode == WNB_MODE_SAMPLING) {
          float uni;
          if (p.uniforms) {
            uni = p.uniforms[(size_t)min(u0 + u, p.B - 1) * p.max_n + min(i, p.i_last)];
          } else {
            uint32_t rr[4];
            philox4x32_10s((uint32_t)i, (uint32_t)(u0 + u), 0u, 0u, (uint32_t)p.seed, (uint32_t)(p.seed >> 32), rr);
            uni = (float)(rr[0] >> 8) * (1.0f / 16777216.0f);
          }
          float lsum = 0.f;
          int lnz = -1;
          for (int q = q0; q < q1; q++) {
            const float e = expf(lg[q] - best);
            lsum += e;
            if (e > 0.f) lnz = q;
          }
          float incl = lsum;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const float v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          pick = sample_pick(incl, lsum, lnz, uni, lane, [&](float start, float target) {   // (common.cuh)
            float c = start;
            for (int q = q0; q < q1; q++) {
              const float e = expf(lg[q] - best);
              c += e;
              if (c > target && e > 0.f) return q;
            }
            return -1;
          });
        }
        if (lane == 0 && u0 + u < p.B && i < s_n[u]) p.xs[(size_t)(u0 + u) * stride_xs + pos + 1] = pick;
      }
      cons_sync();
    }
  }
}

static size_t stream_work_floats(int NU, int R, int S, int Qp, int Ap, int ks, int L, int O1, int Os, int Sp) {
  const int K1 = ks * R + Ap;
  size_t omax = 1024;  // parts * O <= 1024 floats whenever O/4 <= 256 lanes
  (void)O1; (void)Os; (void)Sp;
  return (size_t)NU * (K1 + 2 * R + 2 * S + Qp + Ap + (size_t)(ks - 1) * L * R + omax);
}

// The streaming kernel's coverage and shared-memory rule: every padded width fits the consumer threads and a ring chunk,
// L <= kMaxLayersS, R, S and Ap are multiples of 4, and the work area of NU utterances plus at least two ring slots fits
// shared memory (NU halves down to 1 until it does).  Returns the ring slots (2 .. 6) with *NU and *work set, or 0 when
// the shape is not covered.
static int stream_plan(int Q, int Ap, int R, int S, int ks, int L, int NU, int* NU_out, size_t* work_out) {
  const int O1 = (2 * R + 3) & ~3, Or = (R + 3) & ~3, Os = (S + 3) & ~3, Sp = Os, Qp = (Q + 3) & ~3;
  const int widths[5] = {O1, Or, Os, Sp, Qp};
  for (int i = 0; i < 5; i++)
    if (widths[i] % 4 != 0 || widths[i] / 4 > kConsThreads || widths[i] * 4 > kChunkBytes) return 0;
  if (L > kMaxLayersS || R % 4 != 0 || S % 4 != 0 || Ap % 4 != 0) return 0;
  size_t work = 0;
  int nslot = 0;
  for (;;) {
    work = stream_work_floats(NU, R, S, Qp, Ap, ks, L, O1, Os, Sp) * sizeof(float);
    const size_t avail = 227 * 1024 - 64 - work - 16 * 16;
    nslot = work + 2 * kChunkBytes + 512 > 227 * 1024 ? 0 : (int)(avail / kChunkBytes);
    if (nslot > 6) nslot = 6;
    if (nslot >= 2 || NU == 1) break;
    NU >>= 1;
  }
  if (nslot < 2) return 0;
  *NU_out = NU;
  *work_out = work;
  return nslot;
}

int decode_stream_supported_shape(int Q, int Ap, int R, int S, int ks, int L) {
  int NU = 1;
  size_t work = 0;
  return Q > 0 && Ap > 0 && R > 0 && S > 0 && ks >= 1 && L >= 1 && stream_plan(Q, Ap, R, S, ks, L, 1, &NU, &work) > 0;
}

// returns WNB_ERR_UNSUPPORTED when the shape does not fit this kernel (the caller may run wnb_decode_at instead)
int decode_stream_launch(StreamParams& p, cudaStream_t st) {
  int NU = 1;
  if (p.B > device_sms() * 2) NU = 4; else if (p.B > device_sms()) NU = 2;
  size_t work = 0;
  const int nslot = stream_plan(p.Q, p.Ap, p.R, p.S, p.ks, p.L, NU, &NU, &work);
  if (nslot < 2) return WNB_ERR_UNSUPPORTED;
  p.nslot = nslot;
  const size_t smem = (size_t)nslot * kChunkBytes + 2 * nslot * sizeof(uint64_t) + work;
  const int grid = cdiv(p.B, NU);
#define WNB_LAUNCH_STREAM(N)                                                                                     \
  do {                                                                                                           \
    WNB_CUDA(cudaFuncSetAttribute(decode_stream_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    decode_stream_kernel<N><<<grid, kStreamThreads, smem, st>>>(p);                                              \
  } while (0)
  if (NU == 4) WNB_LAUNCH_STREAM(4);
  else if (NU == 2) WNB_LAUNCH_STREAM(2);
  else WNB_LAUNCH_STREAM(1);
#undef WNB_LAUNCH_STREAM
  WNB_CHECK_LAUNCH("decode_stream");
  return WNB_OK;
}

}  // namespace wnb

using namespace wnb;

extern "C" {

// Number of floats of the packed decode stream for a configuration (layout in the header comment).
WNB_API size_t wnb_decode_stream_floats(int Q, int Ap, int R, int S, int ks, int L) {
  const size_t O1 = (2 * R + 3) & ~3, Or = (R + 3) & ~3, Os = (S + 3) & ~3, Sp = Os, Qp = (Q + 3) & ~3;
  const size_t K1 = (size_t)ks * R + Ap;
  return (size_t)L * (K1 * O1 + (size_t)R * Or + (size_t)R * Os) + (size_t)S * Sp + (size_t)S * Qp;
}

// 1 when wnb_decode_stream_at covers the configuration, else 0 (no device needed).
WNB_API int wnb_decode_stream_supported(int Q, int Ap, int R, int S, int ks, int L) {
  return decode_stream_supported_shape(Q, Ap, R, S, ks, L);
}

WNB_API int wnb_decode_stream_at(int32_t* xs, const float* h, const float* up_w, const float* up_b, const float* wf,
                                 const float* bf, const float* stream, const float* b1, const float* b2,
                                 const float* bp1, const float* bp2, const int32_t* host_dilations, int L,
                                 void* queues, const int32_t* n_samples, const float* uniforms, float* logits_out,
                                 int B, int P, int max_n, int n_pad, int Th, int Q, int A, int Ap, int R, int S, int ks,
                                 int U, int mode, uint64_t seed, int pos0, int xs_base, int h_frame0,
                                 void* stream_handle) {
  WNB_REQUIRE(B > 0 && P >= 1 && max_n >= 1 && Th >= 1 && Q > 0 && A > 0 && Ap >= A && R > 0 && S > 0 && ks >= 1 &&
                  U >= 0 && L >= 1, "decode_stream: bad shape");
  WNB_REQUIRE(xs && h && wf && bf && stream && b1 && b2 && bp1 && bp2 && n_samples && (queues || ks == 1),
              "decode_stream: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode_stream: U>0 needs upsampling weight and bias");
  WNB_REQUIRE(mode == WNB_MODE_ARGMAX || mode == WNB_MODE_SAMPLING, "decode_stream: mode should be sampling or argmax");
  WNB_REQUIRE(Ap % 4 == 0, "decode_stream: Ap must be a multiple of 4");
  StreamParams p{};
  p.xs = xs; p.h = h; p.up_w = up_w; p.up_b = up_b; p.wf = wf; p.bf = bf; p.b1 = b1; p.b2 = b2; p.bp1 = bp1;
  p.bp2 = bp2; p.stream = stream; p.queues = (float*)queues; p.n_samples = n_samples; p.uniforms = uniforms;
  p.logits_out = logits_out;
  p.B = B; p.P = P; p.max_n = max_n; p.n_pad = n_pad; p.Th = Th; p.Q = Q; p.A = A; p.Ap = Ap; p.R = R; p.S = S;
  p.ks = ks; p.U = U; p.mode = mode; p.L = L; p.seed = seed;
  DecodeWindow win;
  if (!decode_window("decode_stream", P, n_pad, U, ks, max_n, Th, pos0, xs_base, h_frame0, &win)) return WNB_ERR_INVALID;
  p.pos0 = win.pos0; p.i0 = win.i0; p.i_last = win.i_last; p.h_last = win.h_last; p.stride_xs = win.stride_xs;
  p.xs = shift_ptr(xs, -(long long)xs_base); p.h = shift_ptr(h, -(long long)h_frame0);
  p.uniforms = shift_ptr(uniforms, -(long long)win.i0); p.logits_out = shift_ptr(logits_out, -(long long)win.i0 * Q);
  p.O1 = (2 * R + 3) & ~3; p.Or = (R + 3) & ~3; p.Os = (S + 3) & ~3; p.Sp = p.Os; p.Qp = (Q + 3) & ~3;
  const long long K1 = (long long)ks * R + Ap;
  p.off_w2res = K1 * p.O1;
  p.off_w2skip = p.off_w2res + (long long)R * p.Or;
  p.layer_stride = p.off_w2skip + (long long)R * p.Os;
  p.off_p1 = (long long)L * p.layer_stride;
  p.off_p2 = p.off_p1 + (long long)S * p.Sp;
  if (L > kMaxLayersS) {
    set_error("decode_stream: more than %d layers", kMaxLayersS);
    return WNB_ERR_UNSUPPORTED;
  }
  long long off = 0;
  for (int l = 0; l < L; l++) {
    p.dil[l] = host_dilations[l];
    p.qoff[l] = off;
    off += (long long)(ks - 1) * host_dilations[l] * R;
  }
  p.q_per_utt = off;
  int rc = decode_stream_launch(p, (cudaStream_t)stream_handle);
  if (rc == WNB_ERR_UNSUPPORTED) set_error("decode_stream: shape not covered by the streaming kernel");
  return rc;
}

}  // extern "C"
