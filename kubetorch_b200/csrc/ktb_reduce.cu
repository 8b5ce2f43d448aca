// ktb_reduce.cu — gather-reduce variant of the mapped call: out = sum_i op(x_i).
//
// In the reference each rank returns `op(shard).sum()` and the caller receives a list of
// per-rank scalars (kt/serving/spmd/spmd_supervisor.py:547-570) which user code then sums.
// Here rank r reduces its shard in one launch (per-thread accumulators → warp-shuffle tree →
// shared memory across warps → one partial per CTA → last-arriving CTA folds the partials in
// fixed order) and stores the scalar straight into the root's partials[r] (peer store).
//
// HBM-bound: algorithmic bytes = n * sizeof(elem) (read once; the output is 4–8 bytes).
#include "ktb_common.cuh"

#include <algorithm>

namespace ktb {

constexpr int kRedThreads = 256;
constexpr int kRedMaxGrid = 4096;  // per-CTA partials: the last CTA folds them in ONE round of 8 x 16-byte loads per thread
constexpr size_t kRedHeader = 64;  // counter lives in the first 64 bytes of the workspace
int g_red_ctas_per_sm = 4;         // ktb_set_tuning key 6: grid cap in units of 1024 CTAs (<= kRedMaxGrid)
int g_red_loads = 8;               // ktb_set_tuning key 13: 256-bit loads in flight per thread (8 = 64 KiB tile per CTA, default; 4 = 32 KiB)

template <int DT>
struct Acc {
  using type = float;
};
template <>
struct Acc<KTB_I32> {
  using type = long long;
};
template <>
struct Acc<KTB_I64> {
  using type = long long;
};

template <int DT, int OP>
__device__ __forceinline__ typename Acc<DT>::type elem_value(const uint8_t* p, const MapParams& mp) {
  if constexpr (DT == KTB_F32) {
    return apply_f32<OP>(*reinterpret_cast<const float*>(p), mp);
  } else if constexpr (DT == KTB_BF16) {
    uint16_t h = *reinterpret_cast<const uint16_t*>(p);
    return apply_bf16_as_f32<OP>(__uint_as_float((uint32_t)h << 16), mp);
  } else if constexpr (DT == KTB_F16) {
    return apply_f16_as_f32<OP>(__half2float(*reinterpret_cast<const __half*>(p)), mp);
  } else if constexpr (DT == KTB_I32) {
    return (long long)(int)apply_i32<OP>(*reinterpret_cast<const uint32_t*>(p), mp);
  } else {
    return (long long)apply_i64<OP>(*reinterpret_cast<const unsigned long long*>(p), mp);
  }
}

// Sum of the op-mapped elements held in NW 32-bit words.
template <int DT, int OP, int NW>
__device__ __forceinline__ typename Acc<DT>::type words_value(const uint32_t (&w)[NW], const MapParams& mp) {
  if constexpr (DT == KTB_F32) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NW; ++i) s += apply_f32<OP>(__uint_as_float(w[i]), mp);
    return s;
  } else if constexpr (DT == KTB_BF16) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      s += apply_bf16_as_f32<OP>(__uint_as_float(w[i] << 16), mp);
      s += apply_bf16_as_f32<OP>(__uint_as_float(w[i] & 0xffff0000u), mp);
    }
    return s;
  } else if constexpr (DT == KTB_F16) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      s += apply_f16_as_f32<OP>(f.x, mp);
      s += apply_f16_as_f32<OP>(f.y, mp);
    }
    return s;
  } else if constexpr (DT == KTB_I32) {
    long long s = 0;
#pragma unroll
    for (int i = 0; i < NW; ++i) s += (long long)(int)apply_i32<OP>(w[i], mp);
    return s;
  } else {
    unsigned long long s = 0;
#pragma unroll
    for (int i = 0; i < NW; i += 2)
      s += apply_i64<OP>(((unsigned long long)w[i + 1] << 32) | w[i], mp);
    return (long long)s;
  }
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum; result valid in thread 0.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem /* >= 32 entries */) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  T r = 0;
  if (warp == 0) {
    r = (lane < (int)(blockDim.x >> 5)) ? smem[lane] : (T)0;
    r = warp_sum(r);
  }
  __syncthreads();
  return r;
}

template <int DT, int OP, int LOADS>
__global__ void __launch_bounds__(kRedThreads)
    map_reduce_kernel(const uint8_t* src, size_t n_elems, MapParams mp, void* out, uint8_t* ws) {
  using A = typename Acc<DT>::type;
  // cross-CTA partials are kept in fp64 for float sums, int64 for integer sums
  using P = typename std::conditional<std::is_same<A, float>::value, double, long long>::type;
  constexpr size_t ES = dtype_size(DT);
  __shared__ P red[32];
  __shared__ bool is_last;

  const size_t n_bytes = n_elems * ES;
  const bool vec_ok = (((uintptr_t)src) & 31) == 0;
  const size_t n_vec = vec_ok ? (n_bytes >> 5) : 0;  // 32-byte packets

  A acc0 = 0, acc1 = 0, acc2 = 0, acc3 = 0;
  const size_t stride = (size_t)gridDim.x * kRedThreads;
  // CTA-contiguous tiles of LOADS x 256 packets (32 or 64 KiB): LOADS independent 256-bit loads in flight per thread,
  // one tile per CTA when the grid covers the input (the hardware scheduler balances the tail), grid-stride beyond
  // kRedMaxGrid.  The four accumulators are filled round-robin so the summation order is fixed for a given LOADS.
  constexpr size_t kTilePackets = (size_t)LOADS * kRedThreads;
  const size_t n_tiles = n_vec / kTilePackets;
  for (size_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const size_t v = t * kTilePackets + threadIdx.x;
    uint32_t w[LOADS][8];
#pragma unroll
    for (int j = 0; j < LOADS; ++j) ldg256_stream(src + ((v + (size_t)j * kRedThreads) << 5), w[j]);
#pragma unroll
    for (int j = 0; j < LOADS; j += 4) {
      acc0 += words_value<DT, OP, 8>(w[j], mp);
      acc1 += words_value<DT, OP, 8>(w[j + 1], mp);
      acc2 += words_value<DT, OP, 8>(w[j + 2], mp);
      acc3 += words_value<DT, OP, 8>(w[j + 3], mp);
    }
  }
  for (size_t v = n_tiles * kTilePackets + (size_t)blockIdx.x * kRedThreads + threadIdx.x; v < n_vec; v += stride) {
    uint32_t w0[8];
    ldg256_stream(src + (v << 5), w0);
    acc0 += words_value<DT, OP, 8>(w0, mp);
  }
  // element tail (everything when the pointer is not 32-byte aligned)
  const size_t tail0 = (n_vec << 5) / ES;
  for (size_t e = tail0 + (size_t)blockIdx.x * kRedThreads + threadIdx.x; e < n_elems; e += stride)
    acc1 += elem_value<DT, OP>(src + e * ES, mp);

  A acc = (acc0 + acc1) + (acc2 + acc3);
  P part = block_sum<P>((P)acc, red);

  unsigned int* counter = reinterpret_cast<unsigned int*>(ws);
  P* partials = reinterpret_cast<P*>(ws + kRedHeader);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = part;
    // one acq_rel RMW instead of fence + atomic + fence: releases this CTA's partial, and for the CTA that draws
    // the last ticket acquires everyone else's (bar.sync below extends that to the other threads of the CTA)
    unsigned int ticket;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(counter) : "memory");
    is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    // fixed-order fold of the per-CTA partials: every thread issues ALL of its (<= 8) 16-byte L2 loads before the
    // first add, so the tail of the launch is one memory round trip instead of one per 256 partials (16 x 16 B would
    // cost 64 registers and halve the occupancy of the streaming phase; 8 keeps the kernel under 48)
    using P2 = typename std::conditional<std::is_same<P, double>::value, double2, longlong2>::type;
    constexpr int kFoldLoads = kRedMaxGrid / (2 * kRedThreads);
    const unsigned int n = gridDim.x;
    P2 v[kFoldLoads];
#pragma unroll
    for (int j = 0; j < kFoldLoads; ++j) {
      const unsigned int i = 2 * threadIdx.x + (unsigned int)j * 2 * kRedThreads;
      v[j].x = 0;
      v[j].y = 0;
      if (i + 1 < n)
        v[j] = __ldcg(reinterpret_cast<const P2*>(&partials[i]));
      else if (i < n)
        v[j].x = __ldcg(&partials[i]);
    }
    P s = 0;
#pragma unroll
    for (int j = 0; j < kFoldLoads; ++j) s += v[j].x + v[j].y;
    s = block_sum<P>(s, red);
    if (threadIdx.x == 0) {
      if constexpr (std::is_same<A, float>::value)
        *reinterpret_cast<float*>(out) = (float)s;
      else
        *reinterpret_cast<long long*>(out) = (long long)s;
      *counter = 0;  // leave the workspace ready for the next call
    }
  }
}

template <typename T, typename P>
__global__ void __launch_bounds__(kRedThreads) reduce_partials_kernel(const T* partials, int n, T* out) {
  __shared__ P red[32];
  P s = 0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) s += (P)partials[i];
  s = block_sum<P>(s, red);
  if (threadIdx.x == 0) out[0] = (T)s;
}

template <int DT, int OP>
static int launch_reduce_typed(int dev, const uint8_t* src, size_t n_elems, const MapParams& p,
                               void* out, void* ws, cudaStream_t stream) {
  (void)dev;
  constexpr size_t ES = dtype_size(DT);
  const int loads = g_red_loads == 4 ? 4 : 8;
  const size_t tile = (size_t)loads * kRedThreads * 32;  // one tile per CTA
  const size_t tiles = (n_elems * ES + tile - 1) / tile;
  const size_t cap = g_red_ctas_per_sm > 0 ? std::min<size_t>((size_t)kRedMaxGrid, (size_t)g_red_ctas_per_sm * 1024) : kRedMaxGrid;
  int grid = (int)std::min<size_t>(std::max<size_t>(tiles, 1), cap);
  if (loads == 8)
    map_reduce_kernel<DT, OP, 8><<<grid, kRedThreads, 0, stream>>>(src, n_elems, p, out, (uint8_t*)ws);
  else
    map_reduce_kernel<DT, OP, 4><<<grid, kRedThreads, 0, stream>>>(src, n_elems, p, out, (uint8_t*)ws);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int launch_map_reduce(int dev, int op, int dtype, const void* src, size_t n_elems, const MapParams& p,
                      void* out, void* workspace, cudaStream_t stream) {
  int rc = check_reducible("ktb_map_reduce_sum", op, dtype);
  if (rc) return rc;
  KTB_REQUIRE(out && workspace, KTB_ERR_ARG, "ktb_map_reduce_sum: null out/workspace");
  KTB_REQUIRE(src || n_elems == 0, KTB_ERR_ARG, "ktb_map_reduce_sum: null src");
  KTB_REQUIRE((((uintptr_t)src) & (dtype_size(dtype) - 1)) == 0, KTB_ERR_ARG, "ktb_map_reduce_sum: src misaligned");
  return dispatch_elementwise<true>(op, dtype, [&](auto dt, auto o) {
    return launch_reduce_typed<dt, o>(dev, static_cast<const uint8_t*>(src), n_elems, p, out, workspace, stream);
  });
}

int launch_reduce_partials(int dev, int dtype, const void* partials, int n, void* out, cudaStream_t stream) {
  (void)dev;
  KTB_REQUIRE(partials && out && n > 0, KTB_ERR_ARG, "ktb_reduce_partials: bad arguments");
  KTB_REQUIRE(acc_size(dtype) != 0, KTB_ERR_ARG, "ktb_reduce_partials: dtype %d not reducible", dtype);
  if (acc_size(dtype) == 4)
    reduce_partials_kernel<float, double><<<1, kRedThreads, 0, stream>>>((const float*)partials, n, (float*)out);
  else
    reduce_partials_kernel<long long, long long>
        <<<1, kRedThreads, 0, stream>>>((const long long*)partials, n, (long long*)out);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

}  // namespace ktb

using namespace ktb;

extern "C" {

size_t ktb_reduce_workspace_bytes(void) { return kRedHeader + sizeof(double) * kRedMaxGrid; }

int ktb_map_reduce_sum(int dev, int op, int dtype, const void* src, size_t n_elems, double alpha,
                       double beta, void* out, void* workspace, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_GUARD(dev);
  return launch_map_reduce(dev, op, dtype, src, n_elems, make_params(alpha, beta, dtype), out, workspace,
                           reinterpret_cast<cudaStream_t>(stream));
}

int ktb_reduce_partials(int dev, int dtype, const void* partials, int n, void* out, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_GUARD(dev);
  return launch_reduce_partials(dev, dtype, partials, n, out, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
