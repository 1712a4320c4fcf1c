// decode_bf16_park.cu -- parking a stream of a bf16 decode pool (nets/wavenet.py::DecodePool with park_below): its
// dilation queues leave its pool row for a compact store of its own, and later go back into any free row.
//
// A pool row holds layer l's x_l of pool step g in slot g mod qlen, qlen = (ks-1) d_l, each slot a row of the decoder's
// swizzled [64 rows][64 ch] bf16 tiles (db::act_off).  A store holds x_l of the stream's own position v in slot
// v mod qlen, as plain [sum_l qlen_l slots][R] bf16: the convention the prefill leaves in an admission workspace.  So a
// stream whose next position v is the pool's step g parks with the rotation v - g (row slot s -> store slot
// (s + v - g) mod qlen), and resumes at step g' with g' - v, the transplant's rotation.  A store does not depend on g, so
// a counter rebase leaves it alone and the stream can resume into any row of any cluster.  Both kernels copy 16-byte
// units bit for bit; every slot of the row or store is written.
#include "decode_bf16_common.cuh"

namespace wnb {
namespace dpark {

constexpr int kMaxL = 64;
constexpr int kMaxRows = db::kM;   // rows one launch moves

struct ParkParams {
  unsigned char* queues;           // the pool's workspace (B = capacity)
  int bc, units, L;                // rows per cluster; 16-byte units of one row of one slot (R / 8); layers
  long long q_cluster, slot_bytes; // bytes of one cluster's queues, of one slot of the pool (R / 64 tiles)
  long long qslot[kMaxL + 1];      // first slot of layer l; qslot[L] = slots of a store
  unsigned char* store[kMaxRows];
  int slot[kMaxRows], rot[kMaxRows];   // pool row; rotation from source slots to destination slots, any sign
};

// grid (x, row i): every 16-byte unit of every slot of every layer of row i.  kPark: pool row -> store; else store -> row.
template <bool kPark>
__global__ void __launch_bounds__(256) park_kernel(const ParkParams p) {
  const int i = blockIdx.y;
  const int row = p.slot[i] % p.bc;
  unsigned char* q = p.queues + (size_t)(p.slot[i] / p.bc) * p.q_cluster;
  unsigned char* st = p.store[i];
  const long long total = p.qslot[p.L] * p.units;
  const long long store_slot = (long long)p.units * 16;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long S = e / p.units;   // slot of the store layout, over every layer
    const int ch = 8 * (int)(e - S * p.units);
    int l = 0;
    for (int step = kMaxL / 2; step > 0; step >>= 1)   // the last layer whose first slot is <= S
      if (l + step < p.L && p.qslot[l + step] <= S) l += step;
    const long long q0 = p.qslot[l];
    const int qlen = (int)(p.qslot[l + 1] - q0);
    const int s = (int)(S - q0);
    const int t = (int)((s + ((long long)p.rot[i] % qlen + qlen)) % qlen);
    if (kPark) {
      const uint4 v = *reinterpret_cast<const uint4*>(q + (size_t)(q0 + s) * p.slot_bytes + db::act_off(row, ch));
      *reinterpret_cast<uint4*>(st + (size_t)(q0 + t) * store_slot + 2 * ch) = v;
    } else {
      const uint4 v = *reinterpret_cast<const uint4*>(st + (size_t)(q0 + s) * store_slot + 2 * ch);
      *reinterpret_cast<uint4*>(q + (size_t)(q0 + t) * p.slot_bytes + db::act_off(row, ch)) = v;
    }
  }
}

static int grid_for(long long total) {
  const long long g = (total + 255) / 256;
  return (int)(g < 4096 ? (g > 0 ? g : 1) : 4096);
}

// the checks and the launch of both directions; `what` names the entry point in errors
static int park_launch(bool park, const char* what, void* queues, int capacity, const int32_t* slots,
                       void* const* stores, const int32_t* rotations, int n, int R, int ks,
                       const int32_t* host_dilations, int L, void* stream_handle) {
  WNB_REQUIRE(capacity > 0 && n >= 1 && n <= kMaxRows && R > 0 && R % 64 == 0 && ks >= 2 && L >= 1 && L <= kMaxL,
              "%s: bad shape", what);
  WNB_REQUIRE(queues && slots && stores && rotations && host_dilations, "%s: null pointer", what);
  ParkParams p{};
  for (int i = 0; i < n; i++) {
    WNB_REQUIRE(stores[i], "%s: null pointer (store %d)", what, i);
    WNB_REQUIRE(((uintptr_t)stores[i] & 15) == 0, "%s: store %d is not 16-byte aligned", what, i);
    WNB_REQUIRE(slots[i] >= 0 && slots[i] < capacity, "%s: row %d: slot %d of %d", what, i, slots[i], capacity);
    for (int k = 0; k < i; k++) WNB_REQUIRE(slots[k] != slots[i], "%s: slot %d given twice", what, slots[i]);
    p.store[i] = (unsigned char*)stores[i];
    p.slot[i] = slots[i];
    p.rot[i] = rotations[i];
  }
  long long nslots = 0;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(host_dilations[l] >= 1, "%s: dilations must be positive", what);
    p.qslot[l] = nslots;
    nslots += (long long)(ks - 1) * host_dilations[l];
  }
  p.qslot[L] = nslots;
  int ncl;
  db_split(capacity, &ncl, &p.bc);
  p.queues = (unsigned char*)queues;
  p.L = L;
  p.units = R / 8;
  p.q_cluster = (long long)wnb_decode_bf16_workspace(1, R, ks, host_dilations, L);   // one cluster
  p.slot_bytes = (long long)(R / 64) * db::kTile;
  const dim3 grid((unsigned)grid_for(nslots * p.units), (unsigned)n);
  if (park)
    park_kernel<true><<<grid, 256, 0, (cudaStream_t)stream_handle>>>(p);
  else
    park_kernel<false><<<grid, 256, 0, (cudaStream_t)stream_handle>>>(p);
  WNB_CHECK_LAUNCH(what);
  return WNB_OK;
}

}  // namespace dpark
}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API size_t wnb_decode_bf16_park_bytes(int R, int ks, const int32_t* host_dilations, int L) {
  if (R < 1 || ks < 2 || L < 1 || !host_dilations) return 0;
  size_t slots = 0;
  for (int l = 0; l < L; l++) {
    if (host_dilations[l] < 1) return 0;
    slots += (size_t)(ks - 1) * host_dilations[l];
  }
  return slots * (size_t)R * 2;
}

WNB_API int wnb_decode_bf16_pool_park(const void* queues, int capacity, const int32_t* slots, void* const* stores,
                                      const int32_t* rotations, int n, int R, int ks, const int32_t* host_dilations,
                                      int L, void* stream_handle) {
  return dpark::park_launch(true, "decode_bf16_pool_park", const_cast<void*>(queues), capacity, slots, stores,
                            rotations, n, R, ks, host_dilations, L, stream_handle);
}

WNB_API int wnb_decode_bf16_pool_unpark(const void* const* stores, void* queues, int capacity, const int32_t* slots,
                                        const int32_t* rotations, int n, int R, int ks, const int32_t* host_dilations,
                                        int L, void* stream_handle) {
  return dpark::park_launch(false, "decode_bf16_pool_unpark", queues, capacity, slots, const_cast<void* const*>(stores),
                            rotations, n, R, ks, host_dilations, L, stream_handle);
}

}  // extern "C"
