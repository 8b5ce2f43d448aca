// ktb_common.cuh — shared host/device helpers for libktb200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <string>
#include <string.h>
#include <type_traits>

#include "../../include/ktb200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libktb200 is written for sm_90a (H100) only"
#endif

namespace ktb {

// ---- error plumbing ------------------------------------------------------------------------
void set_error(const char* fmt, ...);   // thread-local message (ktb_runtime.cu)

#define KTB_CK(call)                                                                          \
  do {                                                                                        \
    cudaError_t _e = (call);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::ktb::set_error("%s failed at %s:%d: %s (%s)", #call, __FILE__, __LINE__,              \
                       cudaGetErrorName(_e), cudaGetErrorString(_e));                         \
      return KTB_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

#define KTB_REQUIRE(cond, code, ...)                                                          \
  do {                                                                                        \
    if (!(cond)) {                                                                            \
      ::ktb::set_error(__VA_ARGS__);                                                          \
      return (code);                                                                          \
    }                                                                                         \
  } while (0)

// Saves and restores the calling thread's current device (PyTorch shares the thread).
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int dev) {
    err = cudaGetDevice(&prev);
    // always bind: on a fresh host thread cudaGetDevice reports 0 without making a context current, and
    // driver entry points (cuTensorMapEncodeTiled) need a current context
    if (err == cudaSuccess) err = cudaSetDevice(dev);
    ok = (err == cudaSuccess);
  }
  ~DeviceGuard() {
    if (prev >= 0) {
      int cur = -1;
      if (cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
    }
  }
};

#define KTB_GUARD(dev)                                                                        \
  ::ktb::DeviceGuard _guard(dev);                                                             \
  if (!_guard.ok) {                                                                           \
    ::ktb::set_error("cudaSetDevice(%d) failed: %s", (dev), cudaGetErrorString(_guard.err));  \
    return KTB_ERR_CUDA;                                                                      \
  }

// Registered-device table (ktb_runtime.cu).
struct DeviceInfo {
  bool registered = false;
  int sm_count = 0;
  cudaStream_t stream_h2d = nullptr, stream_exec = nullptr, stream_d2h = nullptr;  // host pipeline
  cudaStream_t stream_rank = nullptr;                                              // multi-GPU default
  cudaStream_t stream_stage = nullptr;                                             // staged MLP pulls
  cudaEvent_t host_ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // host pipeline
};
constexpr int kMaxDevices = 16;
DeviceInfo* device_info(int dev);   // nullptr when unregistered
int require_device(int dev);        // KTB_OK or error (sets message)

// Bytes per element; 0 = unknown dtype.  constexpr so that kernels can write `constexpr size_t ES = dtype_size(DT)`.
constexpr size_t dtype_size(int dtype) {
  switch (dtype) {
    case KTB_U8: return 1;
    case KTB_F32: return 4;
    case KTB_BF16: return 2;
    case KTB_I32: return 4;
    case KTB_I64: return 8;
    case KTB_F16: return 2;
    default: return 0;
  }
}

// Bytes of a sum of the dtype's elements: fp32 for the float types, int64 for the integers; 0 = not reducible.
constexpr size_t acc_size(int dtype) {
  return (dtype == KTB_F32 || dtype == KTB_BF16 || dtype == KTB_F16) ? 4
         : (dtype == KTB_I32 || dtype == KTB_I64)                    ? 8
                                                                     : 0;
}

// Whether the byte ranges [a, a + an) and [b, b + bn) overlap.
inline bool overlaps(const void* a, size_t an, const void* b, size_t bn) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + bn && y < x + an;
}

// ---- argument checks of the element-wise entry points (KTB_ERR_ARG with a message naming `who`) ----------------
inline int check_dtype(const char* who, int dtype) {
  KTB_REQUIRE(dtype_size(dtype) != 0, KTB_ERR_ARG, "%s: unknown dtype %d", who, dtype);
  return KTB_OK;
}
inline int check_elementwise(const char* who, int op, int dtype) {
  int rc = check_dtype(who, dtype);
  if (rc) return rc;
  KTB_REQUIRE(op >= KTB_OP_IDENTITY && op <= KTB_OP_AFFINE, KTB_ERR_ARG, "%s: unknown op %d", who, op);
  KTB_REQUIRE(dtype != KTB_U8 || op == KTB_OP_IDENTITY, KTB_ERR_ARG, "%s: KTB_U8 supports KTB_OP_IDENTITY only", who);
  return KTB_OK;
}
inline int check_reducible(const char* who, int op, int dtype) {
  KTB_REQUIRE(acc_size(dtype) != 0, KTB_ERR_ARG, "%s: dtype %d not reducible", who, dtype);
  return check_elementwise(who, op, dtype);
}

// ---- runtime (op, dtype) -> kernel instantiation ----------------------------------------------------------------
// Calls f(DT, OP), both as IntC, for an (op, dtype) that check_elementwise (kReduce = false) or check_reducible
// (kReduce = true) accepted, and returns its status.  The map form runs identity of any dtype as a byte copy,
// <KTB_U8, KTB_OP_IDENTITY>, and {F32, BF16, I32, I64, F16} x {SCALE, AFFINE}; the reduce form runs
// {F32, BF16, I32, I64, F16} x {IDENTITY, SCALE, AFFINE}, since a sum reads typed elements even for identity.
template <int V>
using IntC = std::integral_constant<int, V>;
template <bool kReduce = false, class F>
int dispatch_elementwise(int op, int dtype, F&& f) {
  if constexpr (!kReduce)
    if (op == KTB_OP_IDENTITY) return f(IntC<KTB_U8>{}, IntC<KTB_OP_IDENTITY>{});
  auto with_op = [&](auto dt) {
    if constexpr (kReduce)
      if (op == KTB_OP_IDENTITY) return f(dt, IntC<KTB_OP_IDENTITY>{});
    return op == KTB_OP_SCALE ? f(dt, IntC<KTB_OP_SCALE>{}) : f(dt, IntC<KTB_OP_AFFINE>{});
  };
  switch (dtype) {
    case KTB_F32: return with_op(IntC<KTB_F32>{});
    case KTB_BF16: return with_op(IntC<KTB_BF16>{});
    case KTB_I32: return with_op(IntC<KTB_I32>{});
    case KTB_I64: return with_op(IntC<KTB_I64>{});
    case KTB_F16: return with_op(IntC<KTB_F16>{});
  }
  set_error("unsupported dtype/op %d/%d", dtype, op);
  return KTB_ERR_UNSUPPORTED;
}

// Op-math parameters of a mapped callable, passed by value to kernels.
struct MapParams {
  float alpha_f, beta_f;
  long long alpha_i, beta_i;
};
// alpha/beta → op-math parameters with the reference's (torch CPU eager) scalar semantics, measured against the
// reference runtime's recorded results: `x * alpha` keeps alpha in fp32 for bf16/fp16 tensors, but `+ beta` wraps
// the scalar in a tensor of the RESULT dtype first, i.e. beta is rounded to bf16/fp16 before the fp32 add.
inline MapParams make_params(double alpha, double beta, int dtype = KTB_F32) {
  MapParams p;
  p.alpha_f = (float)alpha;
  p.beta_f = (float)beta;
  if (dtype == KTB_BF16) p.beta_f = __bfloat162float(__float2bfloat16_rn(p.beta_f));
  if (dtype == KTB_F16) p.beta_f = __half2float(__float2half_rn(p.beta_f));
  p.alpha_i = (long long)alpha;
  p.beta_i = (long long)beta;
  return p;
}

#ifdef __CUDACC__
// ---- per-element op math (bit-exact with torch eager semantics) ------------------------------
//   F32 : y = fadd_rn(fmul_rn(x, a), b)      — no FMA contraction (torch does two kernels' worth
//                                              of rounding for x*a+b; scale is a single multiply)
//   BF16: op-math in fp32, result rounded to bf16 (RNE) after EACH step, like ATen's bf16 mul/add
//   I32/I64: wrapping two's-complement
template <int OP>
__device__ __forceinline__ float apply_f32(float x, const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY) return x;
  if constexpr (OP == KTB_OP_SCALE) return __fmul_rn(x, p.alpha_f);
  return __fadd_rn(__fmul_rn(x, p.alpha_f), p.beta_f);
}

__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

template <int OP>
__device__ __forceinline__ float apply_bf16_as_f32(float x, const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY) return x;
  if constexpr (OP == KTB_OP_SCALE) return bf16_round(__fmul_rn(x, p.alpha_f));
  return bf16_round(__fadd_rn(bf16_round(__fmul_rn(x, p.alpha_f)), p.beta_f));
}

// Two packed bf16 in one 32-bit word.
template <int OP>
__device__ __forceinline__ uint32_t apply_bf16x2(uint32_t w, const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY) return w;
  float lo = __uint_as_float(w << 16);
  float hi = __uint_as_float(w & 0xffff0000u);
  float ylo = apply_bf16_as_f32<OP>(lo, p);
  float yhi = apply_bf16_as_f32<OP>(hi, p);
  // results are already bf16-representable: take the high halves
  return (__float_as_uint(ylo) >> 16) | (__float_as_uint(yhi) & 0xffff0000u);
}

__device__ __forceinline__ float f16_round(float x) { return __half2float(__float2half_rn(x)); }

template <int OP>
__device__ __forceinline__ float apply_f16_as_f32(float x, const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY) return x;
  if constexpr (OP == KTB_OP_SCALE) return f16_round(__fmul_rn(x, p.alpha_f));
  return f16_round(__fadd_rn(f16_round(__fmul_rn(x, p.alpha_f)), p.beta_f));
}

// Two packed halves in one 32-bit word.
template <int OP>
__device__ __forceinline__ uint32_t apply_f16x2(uint32_t w, const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY) return w;
  const __half2 h = *reinterpret_cast<const __half2*>(&w);
  const float2 f = __half22float2(h);
  const __half2 r = __floats2half2_rn(apply_f16_as_f32<OP>(f.x, p), apply_f16_as_f32<OP>(f.y, p));
  return *reinterpret_cast<const uint32_t*>(&r);
}

template <int OP>
__device__ __forceinline__ uint32_t apply_i32(uint32_t x, const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY) return x;
  if constexpr (OP == KTB_OP_SCALE) return x * (uint32_t)p.alpha_i;
  return x * (uint32_t)p.alpha_i + (uint32_t)p.beta_i;
}

template <int OP>
__device__ __forceinline__ unsigned long long apply_i64(unsigned long long x, const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY) return x;
  if constexpr (OP == KTB_OP_SCALE) return x * (unsigned long long)p.alpha_i;
  return x * (unsigned long long)p.alpha_i + (unsigned long long)p.beta_i;
}

// Apply op to NW 32-bit words held in registers (NW even for I64).
template <int DT, int OP, int NW>
__device__ __forceinline__ void apply_words(uint32_t (&w)[NW], const MapParams& p) {
  if constexpr (OP == KTB_OP_IDENTITY || DT == KTB_U8) {
    return;
  } else if constexpr (DT == KTB_F32) {
#pragma unroll
    for (int i = 0; i < NW; ++i) w[i] = __float_as_uint(apply_f32<OP>(__uint_as_float(w[i]), p));
  } else if constexpr (DT == KTB_BF16) {
#pragma unroll
    for (int i = 0; i < NW; ++i) w[i] = apply_bf16x2<OP>(w[i], p);
  } else if constexpr (DT == KTB_F16) {
#pragma unroll
    for (int i = 0; i < NW; ++i) w[i] = apply_f16x2<OP>(w[i], p);
  } else if constexpr (DT == KTB_I32) {
#pragma unroll
    for (int i = 0; i < NW; ++i) w[i] = apply_i32<OP>(w[i], p);
  } else {  // I64
#pragma unroll
    for (int i = 0; i < NW; i += 2) {
      unsigned long long x = ((unsigned long long)w[i + 1] << 32) | w[i];
      unsigned long long y = apply_i64<OP>(x, p);
      w[i] = (uint32_t)y;
      w[i + 1] = (uint32_t)(y >> 32);
    }
  }
}

// One element at byte address (scalar tails / unaligned fallback).
template <int DT, int OP>
__device__ __forceinline__ void apply_elem(const uint8_t* src, uint8_t* dst, const MapParams& p) {
  if constexpr (DT == KTB_U8) {
    *dst = *src;
  } else if constexpr (DT == KTB_F32) {
    *reinterpret_cast<float*>(dst) = apply_f32<OP>(*reinterpret_cast<const float*>(src), p);
  } else if constexpr (DT == KTB_BF16) {
    uint16_t h = *reinterpret_cast<const uint16_t*>(src);
    float y = apply_bf16_as_f32<OP>(__uint_as_float((uint32_t)h << 16), p);
    *reinterpret_cast<uint16_t*>(dst) = (uint16_t)(__float_as_uint(y) >> 16);
  } else if constexpr (DT == KTB_F16) {
    const __half h = *reinterpret_cast<const __half*>(src);
    *reinterpret_cast<__half*>(dst) = __float2half_rn(apply_f16_as_f32<OP>(__half2float(h), p));
  } else if constexpr (DT == KTB_I32) {
    *reinterpret_cast<uint32_t*>(dst) = apply_i32<OP>(*reinterpret_cast<const uint32_t*>(src), p);
  } else {
    *reinterpret_cast<unsigned long long*>(dst) =
        apply_i64<OP>(*reinterpret_cast<const unsigned long long*>(src), p);
  }
}

// Philox4x32-10 (Random123; the round of curand_philox4x32_x.h): the four words of counter c under key k.  The noise
// of the MLP heads (ktb_mlp.cu) and of the replay sampler (ktb_replay.cu); kubetorch_b200/sampling.py is its twin.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// ---- PTX: streaming vector loads/stores (no L1 allocation; data is touched once) -------------
// A thread owns 32 contiguous bytes per step; sm_90 moves at most 128 bits per access, so each 32-byte step is
// two 128-bit accesses to adjacent addresses (a warp's pair still covers whole 32-byte sectors).  sm_90 gives L2
// eviction priority to a load or store through a cache-policy operand (createpolicy + L2::cache_hint).
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void ldg128(const void* p, uint32_t (&w)[4]) {
  asm volatile("ld.global.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%4];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
               : "l"(p)
               : "memory");
}
__device__ __forceinline__ void stg128(void* p, const uint32_t (&w)[4]) {
  asm volatile("st.global.L1::no_allocate.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(w[0]),
               "r"(w[1]), "r"(w[2]), "r"(w[3])
               : "memory");
}
// read-once / write-once streaming forms: no L1 allocation, first-to-evict in L2
__device__ __forceinline__ void ldg128_stream(const void* p, uint32_t (&w)[4]) {
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.b32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
               : "l"(p), "l"(l2_evict_first_policy())
               : "memory");
}
__device__ __forceinline__ void stg128_stream(void* p, const uint32_t (&w)[4]) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(w[0]),
               "r"(w[1]), "r"(w[2]), "r"(w[3]), "l"(l2_evict_first_policy())
               : "memory");
}
__device__ __forceinline__ void ldg256(const void* p, uint32_t (&w)[8]) {
  ldg128(p, reinterpret_cast<uint32_t(&)[4]>(w[0]));
  ldg128((const uint8_t*)p + 16, reinterpret_cast<uint32_t(&)[4]>(w[4]));
}
__device__ __forceinline__ void stg256(void* p, const uint32_t (&w)[8]) {
  stg128(p, reinterpret_cast<const uint32_t(&)[4]>(w[0]));
  stg128((uint8_t*)p + 16, reinterpret_cast<const uint32_t(&)[4]>(w[4]));
}
__device__ __forceinline__ void ldg256_stream(const void* p, uint32_t (&w)[8]) {
  ldg128_stream(p, reinterpret_cast<uint32_t(&)[4]>(w[0]));
  ldg128_stream((const uint8_t*)p + 16, reinterpret_cast<uint32_t(&)[4]>(w[4]));
}
__device__ __forceinline__ void stg256_stream(void* p, const uint32_t (&w)[8]) {
  stg128_stream(p, reinterpret_cast<const uint32_t(&)[4]>(w[0]));
  stg128_stream((uint8_t*)p + 16, reinterpret_cast<const uint32_t(&)[4]>(w[4]));
}

// ---- PTX: mbarrier + 1-D bulk async copies (TMA engine, no tensor map) ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// global → shared, completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// shared → global, tracked by the thread's bulk async-group
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// ---- in-kernel flag synchronisation of the push pipeline (ktb_push.cu) ------------------------------------------
constexpr unsigned long long kSpinTimeoutNs = 10ull * 1000 * 1000 * 1000;  // 10 s

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Spin until *flag >= want. Returns false on timeout (and records it in *status).  The limit is the u64 that follows
// the status word in the control block (KTB_CTRL_TIMEOUT_NS; 0 = the 10 s default) — read on the slow path only.
__device__ __forceinline__ bool spin_until(const unsigned long long* flag, unsigned long long want,
                                           unsigned int* status) {
  if (ld_acquire_sys(flag) >= want) return true;
  unsigned long long limit =
      *reinterpret_cast<const volatile unsigned long long*>(reinterpret_cast<const char*>(status) + 8);
  if (limit == 0) limit = kSpinTimeoutNs;
  const unsigned long long t0 = globaltimer_ns();
  while (ld_acquire_sys(flag) < want) {
    __nanosleep(200);
    if (globaltimer_ns() - t0 > limit) {
      atomicExch(status, 1u);
      return false;
    }
  }
  return true;
}

#endif  // __CUDACC__

// Layout of a control block (zero-initialised, one per device, ktb_push_control_bytes() long):
//   [   0,  512)  ready[c]  (u64 per chunk, written by the root into the RANK's block)
//   [ 512, 1024)  ack[r]    (u64 per rank, written by rank r into the ROOT's block)
//   [1024, 1028)  ticket    (u32, local)
//   [1032, 1036)  status    (u32, local; nonzero = a spin timed out)
//   [2048, 2560)  chunk_done[seq & 1][c]  (u32 per chunk and call parity, root-local: finished tiles of chunk c)
#define KTB_CTRL_READY 0
#define KTB_CTRL_ACK 512
#define KTB_CTRL_TICKET 1024
#define KTB_CTRL_STATUS 1032
#define KTB_CTRL_TIMEOUT_NS 1040   /* u64 after the status word: spin limit in ns, 0 = 10 s */
#define KTB_CTRL_CHUNK_DONE 2048
#define KTB_PUSH_MAX_CHUNKS 64

// A per-row input pushed with the rows into a rank's staging half (the MLP heads' side inputs): row i of a shard has
// row_bytes bytes at `offset + i·row_bytes` of the half, and on the root at `src + i·row_bytes` (null on the ranks).
// `name` names it in the errors.
struct PushSide {
  const void* src;
  size_t row_bytes, offset, align;
  const char* name;
};

// The side regions of a staging half that holds `rows` rows of `row_bytes` bytes and is `stride` bytes long
// (KTB_ERR_ARG naming `who` otherwise): each starts at or past the rows, ends within the stride, starts at a multiple
// of its alignment and overlaps no earlier region.
inline int check_push_sides(const char* who, const PushSide* sides, int n_sides, size_t rows, size_t row_bytes,
                            size_t stride) {
  for (int k = 0; k < n_sides; ++k) {
    const PushSide& sd = sides[k];
    const size_t n = rows * sd.row_bytes;
    KTB_REQUIRE(sd.offset >= rows * row_bytes, KTB_ERR_ARG, "%s: %s offset %zu overlaps the rows", who, sd.name,
                sd.offset);
    KTB_REQUIRE(sd.offset <= stride && n <= stride - sd.offset, KTB_ERR_ARG,
                "%s: %s offset %zu + %zu exceeds stage_stride", who, sd.name, sd.offset, n);
    KTB_REQUIRE(sd.offset % sd.align == 0, KTB_ERR_ARG, "%s: %s offset %zu must be a multiple of %zu", who, sd.name,
                sd.offset, sd.align);
    for (int o = 0; o < k; ++o)
      KTB_REQUIRE(sd.offset >= sides[o].offset + rows * sides[o].row_bytes || sd.offset + n <= sides[o].offset,
                  KTB_ERR_ARG, "%s: %s overlaps %s", who, sd.name, sides[o].name);
  }
  return KTB_OK;
}


// ---- kernel-launch entry points shared between translation units --------------------------------
// (ktb_map.cu) enqueue dst = op(src) on the current device.
int launch_map(int dev, int op, int dtype, const void* src, void* dst, size_t n_elems,
               const MapParams& p, int variant, cudaStream_t stream);
// (ktb_push.cu) one warp that holds `stream` until *flag >= want (a timeout raises *status), and one that publishes
// *flag = seq once everything before it on `stream` is visible system-wide.
int launch_flag_wait(const unsigned long long* flag, unsigned long long want, unsigned int* status,
                     cudaStream_t stream);
int launch_flag_publish(unsigned long long* flag, unsigned long long seq, cudaStream_t stream);
// (ktb_reduce.cu)
int launch_map_reduce(int dev, int op, int dtype, const void* src, size_t n_elems, const MapParams& p,
                      void* out, void* workspace, cudaStream_t stream);
int launch_reduce_partials(int dev, int dtype, const void* partials, int n, void* out,
                           cudaStream_t stream);

}  // namespace ktb
