// decode_pool.cu -- moving the dilation queues of one utterance of the fp32 decoders (wnb_decode_at, wnb_decode_stream_at,
// wnb_decode_warp_at): the one kernel a decode pool on the fp32 warp decoder needs (nets/wavenet.py::DecodePool).
//
// The three fp32 decoders share one queue layout (wnb_decode_workspace): per utterance a contiguous block of
// [sum_l (ks-1) d_l slots][R] fp32, layer l's slots starting at slot qslot[l], slot t mod (ks-1) d_l holding x_l(t).  That
// block is at once a pool row, a row of an admission prefill's workspace and the store of a parked stream, so admission
// (rotation g_a - (P - 1)), parking (v - g) and resuming (g' - v) are all the same copy: block src[i] -> block dst[i],
// layer l's slot s to slot (s + rot[i]) mod (ks-1) d_l.  16-byte units, bit for bit; every slot of the destination is
// written.  The bf16 pool has kernels of its own (decode_bf16_pool.cu, decode_bf16_park.cu): they address a cluster's
// swizzled tiles, these blocks are plain.
#include "common.cuh"

namespace wnb {
namespace dmove {

constexpr int kMaxL = 64;
// blocks one launch moves.  The pointers travel as kernel parameters: 64 of each kind, the rotations and the layer table
// take 1.8 KB of the 4 KB parameter space, and 64 is the bf16 pool's count per launch too (one admission group), so the
// pool's launches per call are the same on both decoders.  No fixed count lifts the limit altogether; that would need a
// device-side pointer table, i.e. a host-to-device copy in every call.
constexpr int kMaxRows = 64;

struct MoveParams {
  int units, L;                    // 16-byte units of one slot (R / 4); layers
  long long qslot[kMaxL + 1];      // first slot of layer l; qslot[L] = slots of a block
  const float4* src[kMaxRows];
  float4* dst[kMaxRows];
  int rot[kMaxRows];               // rotation from source slots to destination slots, any sign
};

// grid (x, block i): every 16-byte unit of every slot of every layer of block i, read at source slot s and written at
// destination slot (s + rot) mod qlen
__global__ void __launch_bounds__(256) pool_move_kernel(const MoveParams p) {
  const int i = blockIdx.y;
  const float4* src = p.src[i];
  float4* dst = p.dst[i];
  const long long total = p.qslot[p.L] * p.units;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long S = e / p.units;   // slot of the block, over every layer
    const int u = (int)(e - S * p.units);
    int l = 0;
    for (int step = kMaxL / 2; step > 0; step >>= 1)   // the last layer whose first slot is <= S
      if (l + step < p.L && p.qslot[l + step] <= S) l += step;
    const long long q0 = p.qslot[l];
    const long long qlen = p.qslot[l + 1] - q0;
    const long long t = (S - q0 + ((long long)p.rot[i] % qlen + qlen)) % qlen;
    dst[(q0 + t) * p.units + u] = __ldcs(src + e);
  }
}

static int grid_for(long long total) {
  const long long g = (total + 255) / 256;
  return (int)(g < 4096 ? (g > 0 ? g : 1) : 4096);
}

static bool overlaps(const void* a, const void* b, size_t bytes) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + bytes && y < x + bytes;
}

}  // namespace dmove
}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_decode_pool_move(const void* const* src, void* const* dst, const int32_t* rotations, int n, int R,
                                 int ks, const int32_t* host_dilations, int L, void* stream_handle) {
  using namespace dmove;
  WNB_REQUIRE(n >= 1 && n <= kMaxRows && R > 0 && R % 4 == 0 && ks >= 2 && L >= 1 && L <= kMaxL,
              "decode_pool_move: bad shape");
  WNB_REQUIRE(src && dst && rotations && host_dilations, "decode_pool_move: null pointer");
  MoveParams p{};
  long long nslots = 0;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(host_dilations[l] >= 1, "decode_pool_move: dilations must be positive");
    p.qslot[l] = nslots;
    nslots += (long long)(ks - 1) * host_dilations[l];
  }
  p.qslot[L] = nslots;
  const size_t bytes = (size_t)nslots * R * sizeof(float);
  for (int i = 0; i < n; i++) {
    WNB_REQUIRE(src[i] && dst[i], "decode_pool_move: null pointer (block %d)", i);
    WNB_REQUIRE((((uintptr_t)src[i] | (uintptr_t)dst[i]) & 15) == 0, "decode_pool_move: block %d is not 16-byte aligned",
                i);
    for (int k = 0; k < i; k++)
      WNB_REQUIRE(!overlaps(dst[k], dst[i], bytes), "decode_pool_move: destination of block %d given twice (block %d)",
                  i, k);
    for (int k = 0; k < n; k++)   // an in-place rotation, or a source another block overwrites, would race
      WNB_REQUIRE(!overlaps(src[k], dst[i], bytes), "decode_pool_move: destination of block %d overlaps source %d", i, k);
    p.src[i] = (const float4*)src[i];
    p.dst[i] = (float4*)dst[i];
    p.rot[i] = rotations[i];
  }
  p.L = L;
  p.units = R / 4;
  const dim3 grid((unsigned)grid_for(nslots * p.units), (unsigned)n);
  pool_move_kernel<<<grid, 256, 0, (cudaStream_t)stream_handle>>>(p);
  WNB_CHECK_LAUNCH("decode_pool_move");
  return WNB_OK;
}

}  // extern "C"
