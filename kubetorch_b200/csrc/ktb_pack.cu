// ktb_pack.cu — argument/result packing: many tensors <-> one contiguous arena, and the batched
// form of the mapped call (many small calls, one launch).
//
// Replaces the codec the reference runs on every call and again on every rank:
//   pack   : pickle.dumps + base64.b64encode   kt/serving/utils.py:730-749 (_serialize_body)
//   unpack : b64decode + pickle.loads          kt/serving/http_server.py:1768-1822
//   results: the mirror image                  kt/serving/http_server.py:1825-1842, utils.py:787-813
// Tensor leaves never leave HBM: they are gathered into an arena at KTB_PACK_ALIGN-aligned
// offsets by one segmented kernel; the (tiny) offset table travels on the host.
//
// HBM-bound: algorithmic bytes = 2 * sum(nbytes).  A launch carries its segment descriptors
// *in the kernel parameters* (no descriptor upload, graph-capturable): up to kSegSmall in the
// classic 4 KiB parameter space, up to kSegLarge (28 KiB of parameters, CUDA >= 12.1 large
// kernel parameters) when a call has more, so 1024 shards still go out as ONE launch.  Work is
// split into fixed-size tiles across segments so one huge tensor and a thousand tiny ones both
// fill the machine.
#include "ktb_common.cuh"

#include <algorithm>
#include <memory>
#include <vector>

namespace ktb {

constexpr int kSegSmall = 96;             // descriptors per launch in the 4 KiB parameter space
constexpr int kSegLarge = 1024;           // descriptors per launch with large kernel parameters (< 32764 B)
constexpr int kSegThreads = 256;
constexpr uint32_t kSegTile = 32768;      // bytes per CTA work item
int g_seg_large = 1;                      // ktb_set_tuning key 12: 0 = always kSegSmall descriptors per launch

template <int CAP>
struct SegBatch {
  const uint8_t* src[CAP];
  uint8_t* dst[CAP];
  unsigned long long nbytes[CAP];
  uint32_t tile_prefix[CAP + 1];          // tile_prefix[i] = first tile id of segment i
  int n;
};
static_assert(sizeof(SegBatch<kSegSmall>) + sizeof(MapParams) <= 4096, "small batch must fit the classic param space");
static_assert(sizeof(SegBatch<kSegLarge>) + sizeof(MapParams) <= 32764, "large batch must fit CUDA 12.1+ param space");

template <int DT, int OP, int CAP>
__global__ void __launch_bounds__(kSegThreads)
    seg_map_kernel(const __grid_constant__ SegBatch<CAP> b, const __grid_constant__ MapParams p) {
  constexpr size_t ES = dtype_size(DT);
  const uint32_t n_tiles = b.tile_prefix[b.n];
  for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    // binary search: largest i with tile_prefix[i] <= t
    int lo = 0, hi = b.n - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (b.tile_prefix[mid] <= t) lo = mid; else hi = mid - 1;
    }
    const size_t off = (size_t)(t - b.tile_prefix[lo]) * kSegTile;
    const size_t seg_bytes = (size_t)b.nbytes[lo];
    const size_t len = (seg_bytes - off) < (size_t)kSegTile ? (seg_bytes - off) : (size_t)kSegTile;
    const uint8_t* s = b.src[lo] + off;
    uint8_t* d = b.dst[lo] + off;
    const uintptr_t both = ((uintptr_t)s) | ((uintptr_t)d);
    if ((both & 31) == 0) {
      // 256-bit streaming path: a full tile is 1024 packets = 4 per thread, all loads issued first
      const size_t nv = len >> 5;
      size_t v = threadIdx.x;
      for (; v + 3 * kSegThreads < nv; v += 4 * kSegThreads) {
        uint32_t w[4][8];
#pragma unroll
        for (int j = 0; j < 4; ++j) ldg256_stream(s + ((v + j * kSegThreads) << 5), w[j]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          apply_words<DT, OP, 8>(w[j], p);
          stg256_stream(d + ((v + j * kSegThreads) << 5), w[j]);
        }
      }
      for (; v < nv; v += kSegThreads) {
        uint32_t w0[8];
        ldg256_stream(s + (v << 5), w0);
        apply_words<DT, OP, 8>(w0, p);
        stg256_stream(d + (v << 5), w0);
      }
      const size_t tail = nv << 5;
      for (size_t e = threadIdx.x; e < (len - tail) / ES; e += kSegThreads)
        apply_elem<DT, OP>(s + tail + e * ES, d + tail + e * ES, p);
    } else if ((both & 15) == 0) {
      const size_t nv = len >> 4;
      size_t v = threadIdx.x;
      // two 16-byte loads in flight per thread per step
      for (; v + kSegThreads < nv; v += 2 * kSegThreads) {
        uint32_t w0[4], w1[4];
        ldg128(s + (v << 4), w0);
        ldg128(s + ((v + kSegThreads) << 4), w1);
        apply_words<DT, OP, 4>(w0, p);
        apply_words<DT, OP, 4>(w1, p);
        stg128(d + (v << 4), w0);
        stg128(d + ((v + kSegThreads) << 4), w1);
      }
      for (; v < nv; v += kSegThreads) {
        uint32_t w0[4];
        ldg128(s + (v << 4), w0);
        apply_words<DT, OP, 4>(w0, p);
        stg128(d + (v << 4), w0);
      }
      const size_t tail = nv << 4;
      for (size_t e = threadIdx.x; e < (len - tail) / ES; e += kSegThreads)
        apply_elem<DT, OP>(s + tail + e * ES, d + tail + e * ES, p);
    } else {
      for (size_t e = threadIdx.x; e < len / ES; e += kSegThreads)
        apply_elem<DT, OP>(s + e * ES, d + e * ES, p);
    }
  }
}

template <int CAP>
static int launch_seg(int op, int dtype, const SegBatch<CAP>& b, const MapParams& p, cudaStream_t stream) {
  const uint32_t n_tiles = b.tile_prefix[b.n];
  if (n_tiles == 0) return KTB_OK;
  int grid = (int)n_tiles;  // one 32 KiB tile per CTA: the hardware scheduler balances ragged segments
  return dispatch_elementwise(op, dtype, [&](auto dt, auto o) {
    seg_map_kernel<dt, o, CAP><<<grid, kSegThreads, 0, stream>>>(b, p);
    KTB_CK(cudaGetLastError());
    return KTB_OK;
  });
}

// Splits n segments into launches of <= CAP descriptors (and < 2^31 tiles).
template <int CAP>
static int run_segments_cap(int op, int dtype, const void* const* srcs, void* const* dsts,
                            const size_t* nbytes, int n, const MapParams& p, cudaStream_t stream, SegBatch<CAP>& b) {
  const size_t es = (op == KTB_OP_IDENTITY) ? 1 : dtype_size(dtype);
  b.n = 0;
  b.tile_prefix[0] = 0;
  for (int i = 0; i < n; ++i) {
    if (nbytes[i] == 0) continue;
    KTB_REQUIRE(srcs[i] && dsts[i], KTB_ERR_ARG, "segment %d: null pointer with %zu bytes", i, nbytes[i]);
    KTB_REQUIRE((((uintptr_t)srcs[i] | (uintptr_t)dsts[i]) & (es - 1)) == 0 && nbytes[i] % es == 0,
                KTB_ERR_ARG, "segment %d: not aligned to the element size %zu", i, es);
    const size_t tiles = (nbytes[i] + kSegTile - 1) / kSegTile;
    KTB_REQUIRE(tiles < 0x7fffffffULL, KTB_ERR_ARG, "segment %d: %zu bytes is too large", i, nbytes[i]);
    if (b.n == CAP || (size_t)b.tile_prefix[b.n] + tiles >= 0x7fffffffULL) {
      int rc = launch_seg<CAP>(op, dtype, b, p, stream);
      if (rc) return rc;
      b.n = 0;
    }
    b.src[b.n] = static_cast<const uint8_t*>(srcs[i]);
    b.dst[b.n] = static_cast<uint8_t*>(dsts[i]);
    b.nbytes[b.n] = nbytes[i];
    b.tile_prefix[b.n + 1] = b.tile_prefix[b.n] + (uint32_t)tiles;
    ++b.n;
  }
  if (b.n > 0) return launch_seg<CAP>(op, dtype, b, p, stream);
  return KTB_OK;
}

static int run_segments(int dev, int op, int dtype, const void* const* srcs, void* const* dsts,
                        const size_t* nbytes, int n, const MapParams& p, cudaStream_t stream) {
  (void)dev;
  if (n > kSegSmall && g_seg_large) {
    // 28 KiB descriptor block: per-thread scratch, reused across calls (the launch copies it)
    static thread_local std::unique_ptr<SegBatch<kSegLarge>> big;
    if (!big) big.reset(new SegBatch<kSegLarge>());
    return run_segments_cap<kSegLarge>(op, dtype, srcs, dsts, nbytes, n, p, stream, *big);
  }
  SegBatch<kSegSmall> b;
  return run_segments_cap<kSegSmall>(op, dtype, srcs, dsts, nbytes, n, p, stream, b);
}

}  // namespace ktb

using namespace ktb;

extern "C" {

int ktb_pack_layout(const size_t* nbytes, int n, size_t* offsets, size_t* total) {
  KTB_REQUIRE(n >= 0 && (n == 0 || (nbytes && offsets)) && total, KTB_ERR_ARG, "ktb_pack_layout: null argument");
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    offsets[i] = off;
    size_t padded = (nbytes[i] + KTB_PACK_ALIGN - 1) / KTB_PACK_ALIGN * KTB_PACK_ALIGN;
    KTB_REQUIRE(padded >= nbytes[i] && off + padded >= off, KTB_ERR_ARG, "ktb_pack_layout: size overflow");
    off += padded;
  }
  *total = off;
  return KTB_OK;
}

int ktb_pack(int dev, const void* const* srcs, const size_t* nbytes, int n, void* arena,
             size_t arena_bytes, size_t* offsets, int compute_layout, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(n >= 0, KTB_ERR_ARG, "ktb_pack: negative n");
  if (n == 0) return KTB_OK;
  KTB_REQUIRE(srcs && nbytes && offsets && arena, KTB_ERR_ARG, "ktb_pack: null argument");
  size_t total = 0;
  if (compute_layout) {
    rc = ktb_pack_layout(nbytes, n, offsets, &total);
    if (rc) return rc;
  }
  std::vector<void*> dsts((size_t)n);
  for (int i = 0; i < n; ++i) {
    KTB_REQUIRE(offsets[i] <= arena_bytes && nbytes[i] <= arena_bytes - offsets[i], KTB_ERR_ARG,
                "ktb_pack: segment %d (%zu bytes at offset %zu) exceeds the arena (%zu bytes)", i,
                nbytes[i], offsets[i], arena_bytes);
    dsts[(size_t)i] = static_cast<uint8_t*>(arena) + offsets[i];
  }
  KTB_GUARD(dev);
  return run_segments(dev, KTB_OP_IDENTITY, KTB_U8, srcs, dsts.data(), nbytes, n, make_params(1, 0),
                      reinterpret_cast<cudaStream_t>(stream));
}

int ktb_unpack(int dev, const void* arena, const size_t* offsets, const size_t* nbytes, int n,
               void* const* dsts, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(n >= 0, KTB_ERR_ARG, "ktb_unpack: negative n");
  if (n == 0) return KTB_OK;
  KTB_REQUIRE(arena && offsets && nbytes && dsts, KTB_ERR_ARG, "ktb_unpack: null argument");
  std::vector<const void*> srcs((size_t)n);
  for (int i = 0; i < n; ++i) srcs[(size_t)i] = static_cast<const uint8_t*>(arena) + offsets[i];
  KTB_GUARD(dev);
  return run_segments(dev, KTB_OP_IDENTITY, KTB_U8, srcs.data(), dsts, nbytes, n, make_params(1, 0),
                      reinterpret_cast<cudaStream_t>(stream));
}

int ktb_map_batch(int dev, int op, int dtype, const void* const* srcs, void* const* dsts,
                  const size_t* n_elems, int n, double alpha, double beta, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(n >= 0, KTB_ERR_ARG, "ktb_map_batch: negative n");
  if (n == 0) return KTB_OK;
  KTB_REQUIRE(srcs && dsts && n_elems, KTB_ERR_ARG, "ktb_map_batch: null argument");
  rc = check_elementwise("ktb_map_batch", op, dtype);
  if (rc) return rc;
  const size_t es = dtype_size(dtype);
  std::vector<size_t> nb((size_t)n);
  for (int i = 0; i < n; ++i) nb[(size_t)i] = n_elems[i] * es;
  KTB_GUARD(dev);
  return run_segments(dev, op, dtype, srcs, dsts, nb.data(), n, make_params(alpha, beta, dtype),
                      reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
