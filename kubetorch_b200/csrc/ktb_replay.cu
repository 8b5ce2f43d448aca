// ktb_replay.cu — prioritized experience replay, the proportional sampler of include/ktb200.h:
//   ktb_per_sample_f32  builds the sum tree of a priority vector and draws stratified samples and importance weights;
//   ktb_per_update_f32  writes the new priorities (|td| + eps)^alpha in place, the last occurrence of an index winning.
//
// The sampler is stateless: each call builds its tree, in heap order, into the caller's scratch, then draws.
//   blocks  one CTA per 2048 leaves sums them pairwise into the 11 levels of its subtree (registers, shfl.xor, shared
//           memory) and writes their min into tree[blockIdx.x], a slot the next launch overwrites;
//   top     when there is more than one such CTA, one CTA folds their mins and builds the levels above them.  The ABI
//           has no workspace, so there is no zeroed word for a last-CTA ticket: a second launch orders the two;
//   draw    one thread per stratum: one Philox call, then the descent from node 1, log2(P) dependent pairs of loads.
// Every node is one fp32 add of its two children, so the tree is the torch body's level by level whichever lane adds
// (an fp32 a + b is commutative).  About 4·C + 4·P bytes move for the tree.
#include "ktb_common.cuh"

#include <atomic>
#include <cmath>

namespace ktb {

constexpr int kTreeThreads = 256;
constexpr int kTreeLeaves = 8;                           // leaves per thread: levels 1-3 in registers
constexpr int kTreeSpan = kTreeThreads * kTreeLeaves;    // 2048 leaves per CTA: levels 1-11
constexpr int kTopThreads = 1024;
constexpr int kDrawThreads = 128;
constexpr int kUpdateThreads = 1024;
constexpr size_t kPerMaxBatch = 8192;
constexpr size_t kPerMaxC = size_t(1) << 30;
constexpr int kUpdateMaxSmem = 2 * 8192 * 8;             // the hash table at B = 8192: 128 KiB
constexpr uint32_t kEmpty = 0xffffffffu;                 // no valid index (< 2^30) is this key

// torch.min's order: a NaN wins over every number and stays; otherwise the smaller one (fminf would drop the NaN).
__device__ __forceinline__ float nan_min(float m, float x) { return (x < m || x != x) ? x : m; }

// pw(x, s) of include/ktb200.h: torch's pow of an fp32 CUDA tensor by a scalar exponent.  ATen fills 1 at s = 0,
// copies at s = 1, takes sqrt, rsqrt and reciprocal at 0.5, -0.5 and -1, multiplies at 2, 3 and -2 (the last as
// `1.0 / (base * base)`, a double division), and calls powf otherwise.
__device__ __forceinline__ float torch_pow(float x, float s) {
  if (s == 0.0f) return 1.0f;
  if (s == 1.0f) return x;
  if (s == 0.5f) return __fsqrt_rn(x);
  if (s == -0.5f) return rsqrtf(x);
  if (s == -1.0f) return __fdiv_rn(1.0f, x);
  if (s == 2.0f) return __fmul_rn(x, x);
  if (s == 3.0f) return __fmul_rn(__fmul_rn(x, x), x);
  if (s == -2.0f) return (float)(1.0 / (double)__fmul_rn(x, x));
  return powf(x, s);
}

// The internal nodes of one CTA's subtree of kTreeSpan leaves (of all P leaves when P < kTreeSpan) up to its root, node
// P / kTreeSpan + blockIdx.x (node 1 when one CTA covers the tree), and the min of its real leaves in tree[blockIdx.x].
// Node m of level k (level 0 the leaves) is heap node (P >> k) + m, stored when it exists (m < P >> k).
__global__ void __launch_bounds__(kTreeThreads)
    per_tree_blocks_kernel(const float* __restrict__ prio, size_t C, size_t P, float* __restrict__ tree) {
  __shared__ float node8[kTreeThreads / 32], min8[kTreeThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const size_t leaf0 = (size_t)blockIdx.x * kTreeSpan + (size_t)t * kTreeLeaves;
  auto put = [&](int k, size_t m, float v) {
    if (m < (P >> k)) tree[(P >> k) + m] = v;
  };

  float x[kTreeLeaves];
  const float* src = prio + leaf0;
  if (leaf0 + kTreeLeaves <= C && ((uintptr_t)src & 15) == 0) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src) + 1);
    x[0] = a.x, x[1] = a.y, x[2] = a.z, x[3] = a.w, x[4] = b.x, x[5] = b.y, x[6] = b.z, x[7] = b.w;
  } else {
#pragma unroll
    for (int k = 0; k < kTreeLeaves; ++k) x[k] = leaf0 + k < C ? __ldg(src + k) : 0.0f;   // +0 pads to P
  }
  float mn = __int_as_float(0x7f800000);
#pragma unroll
  for (int k = 0; k < kTreeLeaves; ++k)
    if (leaf0 + k < C) mn = nan_min(mn, x[k]);
  if (P == 1 && t == 0) tree[1] = x[0];   // one leaf: it is the root

  float v[kTreeLeaves / 2];
#pragma unroll
  for (int k = 0; k < 4; ++k) put(1, (leaf0 >> 1) + k, v[k] = __fadd_rn(x[2 * k], x[2 * k + 1]));
#pragma unroll
  for (int k = 0; k < 2; ++k) put(2, (leaf0 >> 2) + k, v[k] = __fadd_rn(v[2 * k], v[2 * k + 1]));
  float s = __fadd_rn(v[0], v[1]);
  size_t m = leaf0 >> 3;
  put(3, m, s);
#pragma unroll
  for (int k = 4; k <= 8; ++k) {   // a warp's 32 level-3 nodes
    s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 1 << (k - 4)));
    m >>= 1;
    if ((lane & ((1 << (k - 3)) - 1)) == 0) put(k, m, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if (lane == 0) {
    node8[warp] = s;
    min8[warp] = mn;
  }
  __syncthreads();
  if (warp == 0) {   // the CTA's 8 level-8 nodes, in lanes 0-7 (lanes 8-31 repeat them and store nothing)
    const int w = lane & 7;
    s = node8[w];
    mn = min8[w];
    m = (size_t)blockIdx.x * 8 + w;
#pragma unroll
    for (int k = 9; k <= 11; ++k) {
      s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 1 << (k - 9)));
      mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, 1 << (k - 9)));
      m >>= 1;
      if (lane < 8 && (lane & ((1 << (k - 8)) - 1)) == 0) put(k, m, s);
    }
    if (lane == 0) tree[blockIdx.x] = mn;
  }
}

// The levels above the n >= 2 block roots at tree[n, 2n), and tree[0] = the min of the blocks' mins in tree[0, n).
// Every min is read before the first level overwrites tree[n / 2, n); L1 is bypassed for nodes this CTA wrote.
__global__ void __launch_bounds__(kTopThreads) per_tree_top_kernel(float* __restrict__ tree, size_t n) {
  __shared__ float mins[kTopThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  float mn = __int_as_float(0x7f800000);
  for (size_t i = t; i < n; i += kTopThreads) mn = nan_min(mn, __ldcg(tree + i));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if (lane == 0) mins[warp] = mn;
  __syncthreads();
  for (size_t s = n >> 1; s >= 1; s >>= 1) {
    for (size_t m = t; m < s; m += kTopThreads)
      tree[s + m] = __fadd_rn(__ldcg(tree + 2 * (s + m)), __ldcg(tree + 2 * (s + m) + 1));
    __syncthreads();
  }
  if (warp == 0) {
    mn = mins[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    if (lane == 0) tree[0] = mn;
  }
}

// One thread per stratum j in [j0, j0 + rows): the header's draw, in its order of fp32 operations.
__global__ void __launch_bounds__(kDrawThreads)
    per_draw_kernel(const float* __restrict__ prio, const float* __restrict__ tree, size_t C, size_t P, size_t j0,
                    size_t rows, uint64_t seed, float inv_batch, float c_f, float neg_beta,
                    int64_t* __restrict__ indices, float* __restrict__ weights) {
  const size_t r = (size_t)blockIdx.x * kDrawThreads + threadIdx.x;
  if (r >= rows) return;
  const size_t j = j0 + r;
  const float total = tree[1], mn = tree[0];
  const uint32_t x = philox4x32_10(make_uint4((uint32_t)j, (uint32_t)(j >> 32), 0u, 4u),
                                   make_uint2((uint32_t)seed, (uint32_t)(seed >> 32))).x;
  const float u = (float)(2u * (x >> 9) + 1u) * 5.9604644775390625e-8f;
  float mass = __fmul_rn(__fadd_rn((float)j, u), __fmul_rn(total, inv_batch));
  size_t n = 1;
  while (n < P) {
    const size_t c = 2 * n;
    float left, right;
    if (c < P) {
      left = tree[c];
      right = tree[c + 1];
    } else {   // leaves: the priorities, +0 past C
      left = c - P < C ? prio[c - P] : 0.0f;
      right = c + 1 - P < C ? prio[c + 1 - P] : 0.0f;
    }
    const bool go = mass >= left && right > 0.0f;   // never into a subtree of no mass (a NaN is not > 0)
    if (go) mass = __fsub_rn(mass, left);
    n = c + (go ? 1 : 0);
  }
  const size_t i = n - P;
  indices[r] = (int64_t)i;
  weights[r] = __fdiv_rn(torch_pow(__fmul_rn(__fdiv_rn(prio[i], total), c_f), neg_beta),
                         torch_pow(__fmul_rn(__fdiv_rn(mn, total), c_f), neg_beta));
}

// One CTA: a shared-memory hash table of 2^log2_slots >= 2·B slots maps each index in [0, C) to the largest position
// that holds it (atomicMax: the same whatever order the threads insert in), then the position found there writes.
__global__ void __launch_bounds__(kUpdateThreads)
    per_update_kernel(float* __restrict__ prio, size_t C, const int64_t* __restrict__ indices,
                      const float* __restrict__ td, int B, int log2_slots, float alpha, float eps) {
  extern __shared__ uint32_t slots[];
  const int S = 1 << log2_slots;
  uint32_t* key = slots;
  int* last = reinterpret_cast<int*>(slots + S);
  for (int h = threadIdx.x; h < S; h += kUpdateThreads) {
    key[h] = kEmpty;
    last[h] = -1;
  }
  __syncthreads();
  auto slot_of = [&](uint32_t k, bool insert) {
    uint32_t h = (k * 0x9E3779B1u) >> (32 - log2_slots);
    while (true) {
      const uint32_t old = insert ? atomicCAS(&key[h], kEmpty, k) : key[h];
      if (old == k || (insert && old == kEmpty)) return h;
      h = (h + 1) & (S - 1);
    }
  };
  for (int b = threadIdx.x; b < B; b += kUpdateThreads) {
    const int64_t i = indices[b];
    if (i >= 0 && (uint64_t)i < C) atomicMax(&last[slot_of((uint32_t)i, true)], b);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += kUpdateThreads) {
    const int64_t i = indices[b];
    if (i >= 0 && (uint64_t)i < C && last[slot_of((uint32_t)i, false)] == b)
      prio[i] = torch_pow(__fadd_rn(fabsf(td[b]), eps), alpha);
  }
}

}  // namespace ktb

using namespace ktb;

extern "C" {

int ktb_per_sample_f32(int dev, const float* priorities, size_t C, size_t batch, size_t j0, size_t rows, uint64_t seed,
                       float beta, float* tree, int64_t* indices, float* weights, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(std::isfinite(beta) && beta >= 0.0f, KTB_ERR_ARG, "ktb_per_sample_f32: beta (%g) must be finite and >= 0",
              (double)beta);
  KTB_REQUIRE(C >= 1 && C <= kPerMaxC, KTB_ERR_ARG, "ktb_per_sample_f32: C = %zu must be in [1, 2^30]", C);
  KTB_REQUIRE(batch >= 1, KTB_ERR_ARG, "ktb_per_sample_f32: batch must be >= 1");
  KTB_REQUIRE(batch <= kPerMaxBatch, KTB_ERR_UNSUPPORTED, "ktb_per_sample_f32: batch = %zu is above 8192", batch);
  KTB_REQUIRE(j0 <= batch && rows <= batch - j0, KTB_ERR_ARG,
              "ktb_per_sample_f32: strata [%zu, %zu + %zu) are not inside batch = %zu", j0, j0, rows, batch);
  if (rows == 0) return KTB_OK;
  const void* const ptrs[4] = {priorities, tree, indices, weights};
  const char* const names[4] = {"priorities", "tree", "indices", "weights"};
  for (int k = 0; k < 4; ++k) {
    KTB_REQUIRE(ptrs[k] != nullptr, KTB_ERR_ARG, "ktb_per_sample_f32: %s is NULL", names[k]);
    KTB_REQUIRE(((uintptr_t)ptrs[k] & (k == 2 ? 7 : 3)) == 0, KTB_ERR_ARG, "ktb_per_sample_f32: %s is not %d-byte aligned",
                names[k], k == 2 ? 8 : 4);
  }
  size_t P = 1;
  while (P < C) P <<= 1;
  const size_t bytes[4] = {C * 4, (P < 2 ? 2 : P) * 4, rows * 8, rows * 4};
  for (int o = 1; o < 4; ++o)
    for (int k = 0; k < o; ++k)
      KTB_REQUIRE(!overlaps(ptrs[o], bytes[o], ptrs[k], bytes[k]), KTB_ERR_ARG, "ktb_per_sample_f32: %s overlaps %s",
                  names[o], names[k]);
  KTB_GUARD(dev);
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const size_t blocks = P > (size_t)kTreeSpan ? P / kTreeSpan : 1;
  per_tree_blocks_kernel<<<(unsigned)blocks, kTreeThreads, 0, s>>>(priorities, C, P, tree);
  if (blocks > 1) per_tree_top_kernel<<<1, kTopThreads, 0, s>>>(tree, blocks);
  per_draw_kernel<<<(unsigned)((rows + kDrawThreads - 1) / kDrawThreads), kDrawThreads, 0, s>>>(
      priorities, tree, C, P, j0, rows, seed, 1.0f / (float)batch, (float)C, -beta, indices, weights);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int ktb_per_update_f32(int dev, float* priorities, size_t C, const int64_t* indices, const float* td, size_t B,
                       float alpha, float eps, uintptr_t stream) {
  static std::atomic<unsigned> smem_set{0};   // the devices whose per_update_kernel has opted in to kUpdateMaxSmem
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(std::isfinite(alpha) && std::isfinite(eps), KTB_ERR_ARG,
              "ktb_per_update_f32: alpha (%g) and eps (%g) must be finite", (double)alpha, (double)eps);
  KTB_REQUIRE(C >= 1 && C <= kPerMaxC, KTB_ERR_ARG, "ktb_per_update_f32: C = %zu must be in [1, 2^30]", C);
  KTB_REQUIRE(B >= 1, KTB_ERR_ARG, "ktb_per_update_f32: B must be >= 1");
  KTB_REQUIRE(B <= kPerMaxBatch, KTB_ERR_UNSUPPORTED, "ktb_per_update_f32: B = %zu is above 8192", B);
  const void* const ptrs[3] = {priorities, indices, td};
  const char* const names[3] = {"priorities", "indices", "td"};
  for (int k = 0; k < 3; ++k) {
    KTB_REQUIRE(ptrs[k] != nullptr, KTB_ERR_ARG, "ktb_per_update_f32: %s is NULL", names[k]);
    KTB_REQUIRE(((uintptr_t)ptrs[k] & (k == 1 ? 7 : 3)) == 0, KTB_ERR_ARG, "ktb_per_update_f32: %s is not %d-byte aligned",
                names[k], k == 1 ? 8 : 4);
  }
  KTB_REQUIRE(!overlaps(priorities, C * 4, indices, B * 8), KTB_ERR_ARG, "ktb_per_update_f32: priorities overlaps indices");
  KTB_REQUIRE(!overlaps(priorities, C * 4, td, B * 4), KTB_ERR_ARG, "ktb_per_update_f32: priorities overlaps td");
  KTB_GUARD(dev);
  if (!(smem_set.load(std::memory_order_acquire) & (1u << dev))) {   // dev < kMaxDevices: require_device checked it
    KTB_CK(cudaFuncSetAttribute(per_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kUpdateMaxSmem));
    smem_set.fetch_or(1u << dev, std::memory_order_release);
  }
  int log2_slots = 1;
  while ((size_t(1) << log2_slots) < 2 * B) ++log2_slots;
  per_update_kernel<<<1, kUpdateThreads, (size_t(8) << log2_slots), reinterpret_cast<cudaStream_t>(stream)>>>(
      priorities, C, indices, td, (int)B, log2_slots, alpha, eps);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

}  // extern "C"
