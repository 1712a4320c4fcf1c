// decode_bf16_pool.cu -- the two kernels of a continuous-batching pool on the bf16 decoder (nets/wavenet.py::DecodePool).
//
// A pool runs decode_bf16_kernel unchanged on a batch of `capacity` rows, one launch per call with P = 1, n_pad = 0,
// U = 0 and pos0 = g0, a global step counter shared by every row.  With these arguments the kernel indexes its queue
// slots, xs columns, aux columns and uniforms by g, and each row's inputs are made to mean the right thing for the stream
// that occupies it:
//   * the queues: an admitted stream's warm-up runs through wnb_decode_bf16_prefill into a scratch workspace, and
//     pool_transplant_kernel moves its rows into the pool's workspace.  The warm-up leaves x_l(t) in slot t mod qlen,
//     qlen = (ks-1) d_l, for the last qlen positions before P - 1; the pool's step g_a (the stream's first) plays the
//     part of position P - 1, so slot s goes to (s + g_a - (P - 1)) mod qlen.  Every slot is rewritten (P >= rf gives a
//     full window), so nothing of the row's previous occupant survives;
//   * the aux window and the uniforms: pool_inputs_kernel writes, for every row and every step of the call, the fp32 aux
//     value the decoder would compute in-kernel for that stream's own sample index (fmaf(h[j / U], up_w[j % U], up_b),
//     or h[j] when U = 0), and the Philox uniform of (sample index, stream id), turned into a float as the decoder does.
// Rows of a wgmma product are independent, so each stream's codes are those of one-shot decoding, bit for bit.
#include "decode_bf16_common.cuh"

namespace wnb {
namespace dpool {

constexpr int kMaxL = 64;
constexpr int kMaxRows = db::kM;   // rows one transplant moves: one admission cluster

struct TransplantParams {
  const unsigned char* src; unsigned char* dst;
  int src_bc, dst_bc, units;       // units: 16-byte units of one row of one slot (R / 8)
  long long q_cluster, slot_bytes; // bytes of one cluster's queues, of one slot (R / 64 tiles)
  int qlen[kMaxL];
  long long qslot[kMaxL];          // first slot of layer l
  int src_row[kMaxRows], dst_slot[kMaxRows], rot[kMaxRows];   // rot: g_a - (P - 1), any sign
};

// grid (x, row i, layer l): every 16-byte unit of every slot of layer l of row i
__global__ void __launch_bounds__(256) pool_transplant_kernel(const TransplantParams p) {
  const int i = blockIdx.y, l = blockIdx.z;
  const int qlen = p.qlen[l];
  const int sr = p.src_row[i], dr = p.dst_slot[i];
  const int s_row = sr % p.src_bc, d_row = dr % p.dst_bc;
  const unsigned char* src = p.src + (size_t)(sr / p.src_bc) * p.q_cluster;
  unsigned char* dst = p.dst + (size_t)(dr / p.dst_bc) * p.q_cluster;
  const long long rot = ((long long)p.rot[i] % qlen + qlen) % qlen;
  const long long total = (long long)qlen * p.units;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(e / p.units), ch = 8 * (int)(e - (long long)s * p.units);
    const int t = (int)((s + rot) % qlen);
    const uint4 v = *reinterpret_cast<const uint4*>(src + (size_t)(p.qslot[l] + s) * p.slot_bytes + db::act_off(s_row, ch));
    *reinterpret_cast<uint4*>(dst + (size_t)(p.qslot[l] + t) * p.slot_bytes + db::act_off(d_row, ch)) = v;
  }
}

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
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

// one element per thread: aux[b][a][k] for a < A, uniforms[b][k] for a == A; zero past the row's count
__global__ void __launch_bounds__(256) pool_inputs_kernel(const float* __restrict__ frames, const float* __restrict__ up_w,
                                                          const float* __restrict__ up_b, const int32_t* __restrict__ table,
                                                          float* __restrict__ aux, float* __restrict__ uniforms, int B,
                                                          int A, int F, int n, int U, unsigned long long seed) {
  const long long total = (long long)B * (A + 1) * n;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(e % n);
    const int a = (int)((e / n) % (A + 1));
    const int b = (int)(e / ((long long)n * (A + 1)));
    const bool on = k < table[4 * B + b];
    if (a == A) {
      if (!uniforms) continue;
      float u = 0.f;
      if (on) {
        uint32_t rr[4];
        philox4x32_10((uint32_t)(table[2 * B + b] + k), (uint32_t)table[3 * B + b], 0u, 0u, (uint32_t)seed,
                      (uint32_t)(seed >> 32), rr);
        u = (float)(rr[0] >> 8) * (1.0f / 16777216.0f);
      }
      uniforms[(size_t)b * n + k] = u;
      continue;
    }
    float v = 0.f;
    if (on) {
      const int j = table[B + b] + k;                      // the stream's own aux column
      const int f = (U > 0 ? j / U : j) - table[b];        // its staged frame
      if (f >= 0 && f < F) {
        const float hv = __ldg(frames + ((size_t)b * A + a) * F + f);
        v = U > 0 ? fmaf(hv, __ldg(up_w + j % U), __ldg(up_b)) : hv;
      }
    }
    aux[((size_t)b * A + a) * n + k] = v;
  }
}

static int grid_for(long long total) {
  const long long g = (total + 255) / 256;
  return (int)(g < 4096 ? (g > 0 ? g : 1) : 4096);
}

}  // namespace dpool
}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_decode_bf16_pool_transplant(const void* src_queues, int src_B, const int32_t* src_rows, void* dst_queues,
                                            int capacity, const int32_t* dst_slots, const int32_t* rotations, int n,
                                            int R, int ks, const int32_t* host_dilations, int L, void* stream_handle) {
  using namespace dpool;
  WNB_REQUIRE(src_B > 0 && capacity > 0 && n >= 1 && n <= kMaxRows && R > 0 && R % 64 == 0 && ks >= 2 && L >= 1 &&
                  L <= kMaxL,
              "decode_bf16_pool_transplant: bad shape");
  WNB_REQUIRE(src_queues && dst_queues && src_rows && dst_slots && rotations && host_dilations,
              "decode_bf16_pool_transplant: null pointer");
  TransplantParams p{};
  for (int i = 0; i < n; i++) {
    WNB_REQUIRE(src_rows[i] >= 0 && src_rows[i] < src_B && dst_slots[i] >= 0 && dst_slots[i] < capacity,
                "decode_bf16_pool_transplant: row %d: source row %d of %d, slot %d of %d", i, src_rows[i], src_B,
                dst_slots[i], capacity);
    for (int k = 0; k < i; k++)
      WNB_REQUIRE(dst_slots[k] != dst_slots[i], "decode_bf16_pool_transplant: slot %d given twice", dst_slots[i]);
    p.src_row[i] = src_rows[i];
    p.dst_slot[i] = dst_slots[i];
    p.rot[i] = rotations[i];
  }
  long long slots = 0;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(host_dilations[l] >= 1, "decode_bf16_pool_transplant: dilations must be positive");
    p.qlen[l] = (ks - 1) * host_dilations[l];
    p.qslot[l] = slots;
    slots += p.qlen[l];
  }
  int ncl;
  db_split(src_B, &ncl, &p.src_bc);
  db_split(capacity, &ncl, &p.dst_bc);
  p.q_cluster = (long long)wnb_decode_bf16_workspace(1, R, ks, host_dilations, L);   // one cluster
  p.src = (const unsigned char*)src_queues;
  p.dst = (unsigned char*)dst_queues;
  p.units = R / 8;
  p.slot_bytes = (long long)(R / 64) * db::kTile;
  int maxq = 0;
  for (int l = 0; l < L; l++) maxq = maxq > p.qlen[l] ? maxq : p.qlen[l];
  const int gx = grid_for((long long)maxq * p.units);
  pool_transplant_kernel<<<dim3((unsigned)gx, (unsigned)n, (unsigned)L), 256, 0, (cudaStream_t)stream_handle>>>(p);
  WNB_CHECK_LAUNCH("decode_bf16_pool_transplant");
  return WNB_OK;
}

WNB_API int wnb_decode_bf16_pool_inputs(const float* frames, const float* up_w, const float* up_b, const int32_t* table,
                                        float* aux, float* uniforms, int B, int A, int F, int n, int U, uint64_t seed,
                                        void* stream_handle) {
  using namespace dpool;
  WNB_REQUIRE(B > 0 && A > 0 && F > 0 && n > 0 && U >= 0, "decode_bf16_pool_inputs: bad shape");
  WNB_REQUIRE(frames && table && aux, "decode_bf16_pool_inputs: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode_bf16_pool_inputs: U>0 needs upsampling weight and bias");
  const long long total = (long long)B * (A + 1) * n;
  pool_inputs_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream_handle>>>(frames, up_w, up_b, table, aux, uniforms,
                                                                                B, A, F, n, U, seed);
  WNB_CHECK_LAUNCH("decode_bf16_pool_inputs");
  return WNB_OK;
}

}  // extern "C"
