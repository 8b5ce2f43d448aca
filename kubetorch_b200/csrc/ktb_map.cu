// ktb_map.cu — the element-wise mapped callable ("execute" step of the remote-map path).
//
// Replaces the per-rank user-function execution of kt/serving/http_server.py:1845-1891
// (execute_callable_async) for the closed set of registered ops (identity / scale / affine).
// The same kernels serve as the fused scatter→exec→gather when src/dst are peer-mapped
// pointers into the root GPU's arg/result arenas (ktb_dispatch.cu).
//
// HBM-bound: algorithmic bytes = n*(sizeof in + sizeof out); no data reuse, so the only
// levers are coalesced wide accesses, enough bytes in flight, and a grid that is a multiple
// of the SM count.  Three bit-identical variants:
//   VEC    — 128-bit LDG/STG, 4 loads in flight per thread, one tile per CTA
//   TMA    — cp.async.bulk global→shared ring (mbarrier complete_tx), compute in shared,
//            cp.async.bulk shared→global; one elected thread drives the TMA engine
//   SCALAR — any alignment
#include "ktb_common.cuh"

#include <algorithm>

namespace ktb {

// test hooks of ktb_set_tuning, each defined beside the code it steers
extern int g_red_ctas_per_sm;  // ktb_reduce.cu
extern int g_red_loads;        // ktb_reduce.cu
extern int g_seg_large;        // ktb_pack.cu
extern int g_mlp_chunk_rows;   // ktb_mlp.cu
extern int g_mlp_stage_ce;     // ktb_mlp.cu

constexpr int kVecThreads = 256;
constexpr int kVecBytes = 16;   // 128 bits: sm_90 has no wider per-thread global access
constexpr int kVecUnroll = 4;   // 4 x 128-bit loads in flight per thread = one 16 KiB tile per CTA

constexpr int kTmaStages = 4;         // 4 x 32 KiB ring per CTA, one CTA per SM
constexpr int kTmaStageBytes = 32768;
constexpr int kTmaThreads = 256;

// ---- VEC -----------------------------------------------------------------------------------------
// L1::no_allocate + L2::evict_first loads and stores (the data is touched once).
template <int DT, int OP>
__global__ void __launch_bounds__(kVecThreads)
    map_vec_kernel(const uint8_t* src, uint8_t* dst, size_t n_bytes, MapParams p) {
  constexpr int VB = kVecBytes;
  constexpr int NW = VB / 4;
  constexpr size_t TILE = (size_t)kVecThreads * kVecUnroll * VB;  // bytes per CTA iteration
  constexpr size_t ROW = (size_t)kVecThreads * VB;                // bytes per unrolled step
  const size_t n_full = n_bytes / TILE;

  for (size_t t = blockIdx.x; t < n_full; t += gridDim.x) {
    const size_t off = t * TILE + (size_t)threadIdx.x * VB;
    uint32_t w[kVecUnroll][NW];
#pragma unroll
    for (int j = 0; j < kVecUnroll; ++j) ldg128_stream(src + off + j * ROW, w[j]);
#pragma unroll
    for (int j = 0; j < kVecUnroll; ++j) {
      apply_words<DT, OP, NW>(w[j], p);
      stg128_stream(dst + off + j * ROW, w[j]);
    }
  }

  // Remainder (< TILE bytes): one CTA, bounds-checked vectors then an element tail.
  if (blockIdx.x == (unsigned)(n_full % gridDim.x)) {
    const size_t base = n_full * TILE;
    const size_t n_vec = (n_bytes - base) / VB;
    for (size_t v = threadIdx.x; v < n_vec; v += kVecThreads) {
      uint32_t w[NW];
      ldg128_stream(src + base + v * VB, w);
      apply_words<DT, OP, NW>(w, p);
      stg128_stream(dst + base + v * VB, w);
    }
    constexpr size_t ES = dtype_size(DT);
    const size_t tail = base + n_vec * VB;
    const size_t n_tail = (n_bytes - tail) / ES;
    for (size_t e = threadIdx.x; e < n_tail; e += kVecThreads)
      apply_elem<DT, OP>(src + tail + e * ES, dst + tail + e * ES, p);
  }
}

// ---- SCALAR ------------------------------------------------------------------------------------
template <int DT, int OP>
__global__ void __launch_bounds__(256)
    map_scalar_kernel(const uint8_t* src, uint8_t* dst, size_t n_elems, MapParams p) {
  constexpr size_t ES = dtype_size(DT);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_elems; i += stride)
    apply_elem<DT, OP>(src + i * ES, dst + i * ES, p);
}

// ---- TMA -----------------------------------------------------------------------------------------
// One CTA owns a ring of STAGES shared-memory tiles.  Thread 0 is the TMA driver: it arms
// full[s] with the tile's byte count and issues the bulk load; all threads wait on full[s],
// transform the tile in place (16-byte shared accesses, conflict-free), fence the generic→async
// proxy, and thread 0 issues the bulk store.  A stage is re-armed once the bulk store that
// read it has finished reading (cp.async.bulk.wait_group.read), one iteration later, so
// STAGES-1 loads stay in flight per CTA.
template <int DT, int OP>
__global__ void __launch_bounds__(kTmaThreads)
    map_tma_kernel(const uint8_t* src, uint8_t* dst, size_t n_bytes, MapParams p) {
  constexpr int STAGES = kTmaStages, STAGE_BYTES = kTmaStageBytes, NT = kTmaThreads;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* buf = smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)STAGES * STAGE_BYTES);
  constexpr bool kCompute = !(OP == KTB_OP_IDENTITY || DT == KTB_U8);

  const size_t n16 = n_bytes & ~(size_t)15;  // bulk copies move multiples of 16 bytes
  const size_t n_tiles = (n16 + STAGE_BYTES - 1) / STAGE_BYTES;
  const size_t my_n =
      (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  auto tile_off = [&](size_t k) { return ((size_t)blockIdx.x + k * gridDim.x) * STAGE_BYTES; };
  auto tile_len = [&](size_t k) {
    size_t r = n16 - tile_off(k);
    return (uint32_t)(r < (size_t)STAGE_BYTES ? r : (size_t)STAGE_BYTES);
  };

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (threadIdx.x == 0) {
    const size_t pre = my_n < (size_t)STAGES ? my_n : (size_t)STAGES;
    for (size_t k = 0; k < pre; ++k) {
      const uint32_t len = tile_len(k);
      mbar_expect_tx(&full[k], len);
      bulk_g2s(buf + k * STAGE_BYTES, src + tile_off(k), len, &full[k]);
    }
  }

  if (kCompute || threadIdx.x == 0) {
    for (size_t k = 0; k < my_n; ++k) {
      const int s = (int)(k % STAGES);
      const uint32_t parity = (uint32_t)((k / STAGES) & 1);
      const uint32_t len = tile_len(k);
      mbar_wait(&full[s], parity);
      if constexpr (kCompute) {
        uint4* tile = reinterpret_cast<uint4*>(buf + (size_t)s * STAGE_BYTES);
        const uint32_t nv = len >> 4;
        for (uint32_t v = threadIdx.x; v < nv; v += NT) {
          uint4 q = tile[v];
          uint32_t w[4] = {q.x, q.y, q.z, q.w};
          apply_words<DT, OP, 4>(w, p);
          tile[v] = make_uint4(w[0], w[1], w[2], w[3]);
        }
        fence_proxy_async_smem();  // make generic-proxy writes visible to the bulk store
        __syncthreads();
      }
      if (threadIdx.x == 0) {
        bulk_s2g(dst + tile_off(k), buf + (size_t)s * STAGE_BYTES, len);
        bulk_commit();
        if (k >= 1 && (k - 1 + STAGES) < my_n) {
          bulk_wait_read<1>();  // store of tile k-1 has finished reading its stage
          const size_t kn = k - 1 + STAGES;
          const int sn = (int)((k - 1) % STAGES);
          const uint32_t ln = tile_len(kn);
          mbar_expect_tx(&full[sn], ln);
          bulk_g2s(buf + (size_t)sn * STAGE_BYTES, src + tile_off(kn), ln, &full[sn]);
        }
      }
    }
    if (threadIdx.x == 0) bulk_wait_all<0>();
  }

  // < 16 trailing bytes: element tail by CTA 0.
  if (blockIdx.x == 0) {
    constexpr size_t ES = dtype_size(DT);
    const size_t n_tail = (n_bytes - n16) / ES;
    for (size_t e = threadIdx.x; e < n_tail; e += NT)
      apply_elem<DT, OP>(src + n16 + e * ES, dst + n16 + e * ES, p);
  }
}

// ---- launch plumbing --------------------------------------------------------------------------
template <int DT, int OP>
static int launch_typed(int dev, const uint8_t* src, uint8_t* dst, size_t n_bytes, const MapParams& p, int variant,
                        cudaStream_t stream) {
  const DeviceInfo* di = device_info(dev);
  const size_t n_elems = n_bytes / dtype_size(DT);
  const uintptr_t both = (uintptr_t)src | (uintptr_t)dst;

  if (variant == KTB_VARIANT_AUTO) variant = KTB_VARIANT_VEC;
  // bulk (TMA) and vector paths need 16-byte aligned pointers; ragged shard boundaries fall back
  if (variant == KTB_VARIANT_TMA && (both & 15)) variant = KTB_VARIANT_VEC;
  if (variant == KTB_VARIANT_VEC && (both & 15)) variant = KTB_VARIANT_SCALAR;

  if (variant == KTB_VARIANT_VEC) {
    // one tile per CTA: the hardware scheduler balances the tail
    const size_t tiles = std::max<size_t>(n_bytes / ((size_t)kVecThreads * kVecUnroll * kVecBytes), 1);
    const int grid = (int)std::min<size_t>(tiles, 0x7fffffffULL);
    map_vec_kernel<DT, OP><<<grid, kVecThreads, 0, stream>>>(src, dst, n_bytes, p);
  } else if (variant == KTB_VARIANT_TMA) {
    constexpr size_t smem_bytes = (size_t)kTmaStages * kTmaStageBytes + kTmaStages * sizeof(uint64_t);
    auto kfn = map_tma_kernel<DT, OP>;
    KTB_CK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    const size_t tiles = ((n_bytes & ~(size_t)15) + kTmaStageBytes - 1) / kTmaStageBytes;
    const int grid = (int)std::min<size_t>(std::max<size_t>(tiles, 1), (size_t)di->sm_count);
    kfn<<<grid, kTmaThreads, smem_bytes, stream>>>(src, dst, n_bytes, p);
  } else if (variant == KTB_VARIANT_SCALAR) {
    size_t blocks = (n_elems + 255) / 256;
    int grid = (int)std::min<size_t>(std::max<size_t>(blocks, 1), (size_t)di->sm_count * 8);
    map_scalar_kernel<DT, OP><<<grid, 256, 0, stream>>>(src, dst, n_elems, p);
  } else {
    set_error("ktb_map: unknown variant %d", variant);
    return KTB_ERR_ARG;
  }
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int launch_map(int dev, int op, int dtype, const void* src_, void* dst_, size_t n_elems,
               const MapParams& p, int variant, cudaStream_t stream) {
  const uint8_t* src = static_cast<const uint8_t*>(src_);
  uint8_t* dst = static_cast<uint8_t*>(dst_);
  int rc = check_elementwise("ktb_map", op, dtype);
  if (rc) return rc;
  if (n_elems == 0) return KTB_OK;
  const size_t es = dtype_size(dtype);
  KTB_REQUIRE(src && dst, KTB_ERR_ARG, "ktb_map: null src/dst with n_elems=%zu", n_elems);
  KTB_REQUIRE((((uintptr_t)src | (uintptr_t)dst) & (es - 1)) == 0, KTB_ERR_ARG,
              "ktb_map: src/dst not aligned to the element size %zu", es);
  KTB_REQUIRE(n_elems <= (SIZE_MAX / 8), KTB_ERR_ARG, "ktb_map: n_elems too large");
  if (src != dst) {
    const uint8_t* se = src + n_elems * es;
    const uint8_t* de = dst + n_elems * es;
    KTB_REQUIRE(se <= dst || de <= src, KTB_ERR_ARG, "ktb_map: src and dst partially overlap");
  }

  return dispatch_elementwise(op, dtype, [&](auto dt, auto o) {
    return launch_typed<dt, o>(dev, src, dst, n_elems * es, p, variant, stream);
  });
}

}  // namespace ktb

using namespace ktb;

extern "C" {

// Test hooks (not part of the stable ABI, not in ktb200.h): each key steers a launch geometry or path
// that the tests compare against the shipped default.
//   key 6:  map_reduce_sum grid cap in units of 1024 CTAs (<= 0: the default, 4)
//   key 8:  MLP rows per chunk (a positive multiple of 128)
//   key 12: 0 = segment maps use only the 96 descriptors of the classic parameter space
//   key 13: map_reduce_sum 256-bit loads per thread and tile (4, otherwise 8)
//   key 22: 1 = staged MLP pulls by copy engine instead of a pull kernel
int ktb_set_tuning(int key, int value) {
  switch (key) {
    case 6: g_red_ctas_per_sm = value > 0 ? value : 4; return KTB_OK;
    case 12: g_seg_large = value ? 1 : 0; return KTB_OK;
    case 13: g_red_loads = value == 4 ? 4 : 8; return KTB_OK;
    case 22: g_mlp_stage_ce = value ? 1 : 0; return KTB_OK;
    case 8:
      KTB_REQUIRE(value > 0 && value % 128 == 0, KTB_ERR_ARG, "ktb_set_tuning: MLP chunk rows must be a multiple of 128");
      g_mlp_chunk_rows = value;
      return KTB_OK;
    default: set_error("ktb_set_tuning: unknown key %d", key); return KTB_ERR_ARG;
  }
}

int ktb_map(int dev, int op, int dtype, const void* src, void* dst, size_t n_elems, double alpha,
            double beta, int variant, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_GUARD(dev);
  return launch_map(dev, op, dtype, src, dst, n_elems, make_params(alpha, beta, dtype), variant,
                    reinterpret_cast<cudaStream_t>(stream));
}

int ktb_map_identity_u8(int dev, const void* src, void* dst, size_t nbytes, uintptr_t stream) {
  return ktb_map(dev, KTB_OP_IDENTITY, KTB_U8, src, dst, nbytes, 1.0, 0.0, KTB_VARIANT_AUTO, stream);
}
int ktb_map_scale_f32(int dev, const float* src, float* dst, size_t n, float alpha, uintptr_t stream) {
  return ktb_map(dev, KTB_OP_SCALE, KTB_F32, src, dst, n, alpha, 0.0, KTB_VARIANT_AUTO, stream);
}
int ktb_map_affine_f32(int dev, const float* src, float* dst, size_t n, float alpha, float beta,
                       uintptr_t stream) {
  return ktb_map(dev, KTB_OP_AFFINE, KTB_F32, src, dst, n, alpha, beta, KTB_VARIANT_AUTO, stream);
}
int ktb_map_scale_bf16(int dev, const void* src, void* dst, size_t n, float alpha, uintptr_t stream) {
  return ktb_map(dev, KTB_OP_SCALE, KTB_BF16, src, dst, n, alpha, 0.0, KTB_VARIANT_AUTO, stream);
}
int ktb_map_affine_bf16(int dev, const void* src, void* dst, size_t n, float alpha, float beta,
                        uintptr_t stream) {
  return ktb_map(dev, KTB_OP_AFFINE, KTB_BF16, src, dst, n, alpha, beta, KTB_VARIANT_AUTO, stream);
}

}  // extern "C"
