// ktb_mlp.cu — the bf16 MLP policy callable of BASELINE config C4 on Hopper tensor cores (wgmma).
//
// The mapped callable (oracle/cases.py:mlp_policy; what the reference would run per rank inside
// kt/serving/http_server.py:1845-1891) is   logits = W3·relu(W2·relu(W1·obsᵀ))   in bf16.
// It is the one place on this path where the user function is itself a dense GEMM, so it is the
// one place tensor cores are used: each layer is   C[M,N] = act(A[M,K] · B[N,K]ᵀ)   with
//   * A and B tiles staged global→shared by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B, K-major)
//     into a STAGES-deep ring guarded by mbarriers (full: TMA bytes landed, empty: consumers done),
//   * wgmma.mma_async m64nNk16 (bf16 x bf16 → fp32) issued by two consumer warpgroups, each owning
//     64 rows of the 128-row tile, both operands read straight from shared memory by descriptor,
//   * an epilogue from the fp32 register accumulators: optional bias (nn.Linear), fused ReLU + bf16
//     rounding, global stores masked to the head's width, and optionally the greedy action of every
//     row, or instead an action sampled by seeded Gumbel-max with its log-probability — the last
//     layer's outputs may be peer pointers into the root GPU's result arena, which fuses the gather
//     into the epilogue.
// Warp roles (288 threads): warps 0-7 = two consumer warpgroups, warp 8 = TMA producer (one lane).
// Activations are rounded to bf16 between layers (like the eager torch module); rows are processed
// in chunks whose hidden activations stay resident in the 50 MB L2.  One kernel
// (mlp_layer_wgmma_kernel) runs every layer of every entry point.
#include "ktb_common.cuh"

#include <cuda.h>
#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <mutex>

namespace ktb {

constexpr int kMlpBlockM = 128;
constexpr int kMlpBlockK = 64;   // 64 bf16 = 128 bytes = one SWIZZLE_128B row
constexpr int kMlpWgmmaK = 16;
constexpr int kMlpStages = 4;
constexpr int kMlpConsumers = 256;             // two warpgroups
constexpr int kMlpThreads = kMlpConsumers + 32;
int g_mlp_chunk_rows = 16896;  // ktb_set_tuning key 8: rows per chunk = 132 SMs x 128 rows, so each 256-wide layer of a
                               // chunk is four whole waves of 128 x 256 tiles, and one chunk's hidden activation
                               // (34.6 MB at d_hidden = 1024) stays in the 50 MB L2 between the layers

// ---- PTX wrappers -----------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::
          "r"(smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma:
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (unused for swizzled K-major, 1) | [32,46) SBO >> 4
//   [49,52) base offset (0: tiles are 1024-byte aligned) | [62,64) layout type = 1 (SWIZZLE_128B)
// SBO = 1024 bytes: 8 rows x 128 bytes per swizzle atom, atoms stacked along M/N.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(const void* smem_tile) {
  const uint32_t addr = smem_u32(smem_tile);
  uint64_t d = 0;
  d |= (uint64_t)((addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// D[64 x N] (+)= A[64 x 16] · B[N x 16]ᵀ for one warpgroup, fp32 accumulators in registers (N/2 per thread).
template <int N>
struct Wgmma;
template <>
struct Wgmma<256> {
  __device__ __forceinline__ static void mma(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, "
        "%128, %129, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};

template <>
struct Wgmma<128> {
  __device__ __forceinline__ static void mma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
        "%64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};

template <>
struct Wgmma<64> {
  __device__ __forceinline__ static void mma(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
        "%32, %33, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <int BLOCK_N, int STAGES>
struct MlpSmem {
  static constexpr int kABytes = kMlpBlockM * kMlpBlockK * 2;   // 16 KiB
  static constexpr int kBBytes = BLOCK_N * kMlpBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarrierOff = STAGES * kStageBytes;
  static constexpr int kTotal = kBarrierOff + 2 * STAGES * 8 + 1024 /* alignment slack */;
};

// The main loop of an MLP layer: the fp32 tile A[m0:m0+128, :K] · B[n0:n0+BLOCK_N, :K]ᵀ.  The TMA
// producer (warp 8, one lane) fills the STAGES-deep ring and then returns false; each consumer thread returns true
// with its warpgroup's 64 x BLOCK_N accumulators in acc.  A has `rows` rows (the outer dimension of map_a) and B has
// N rows: TMA zero-fills the rows of a box past either end (and still counts the whole box toward complete_tx), so
// the accumulators of those rows and columns are 0 and the epilogue decides what to store.
template <int BLOCK_N, int STAGES>
__device__ __forceinline__ bool mlp_tile_mainloop(const CUtensorMap* map_a, const CUtensorMap* map_b, int K, int m0,
                                                  int n0, float (&acc)[BLOCK_N / 2]) {
  using S = MlpSmem<BLOCK_N, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles must be 1024-byte aligned
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::kBarrierOff);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = K / kMlpBlockK;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kMlpConsumers);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kMlpConsumers / 32) {
    // ===== TMA producer =====
    if (lane == 0) {
      prefetch_tensormap(map_a);
      prefetch_tensormap(map_b);
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        mbar_wait(&empty[s], ((kb / STAGES) & 1) ^ 1);
        uint8_t* a_dst = smem + (size_t)s * S::kStageBytes;
        mbar_expect_tx(&full[s], S::kStageBytes);
        tma_load_2d(a_dst, map_a, kb * kMlpBlockK, m0, &full[s]);
        tma_load_2d(a_dst + S::kABytes, map_b, kb * kMlpBlockK, n0, &full[s]);
      }
    }
    return false;
  }

  // ===== consumer warpgroup wg: rows 64*wg .. 64*wg+63 of the tile =====
  const int wg = warp >> 2;
#pragma unroll
  for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(&full[s], (kb / STAGES) & 1);
    const uint8_t* a_src = smem + (size_t)s * S::kStageBytes + wg * 64 * 128;
    const uint64_t adesc = make_smem_desc_sw128(a_src);
    const uint64_t bdesc = make_smem_desc_sw128(smem + (size_t)s * S::kStageBytes + S::kABytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kMlpBlockK / kMlpWgmmaK; ++k) {
      // advance 16 bf16 = 32 bytes along K inside the 128-byte swizzle row: +2 in the >>4 address field
      Wgmma<BLOCK_N>::mma(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
    }
    wgmma_commit();
    wgmma_wait_all();
    mbar_arrive(&empty[s]);   // this thread no longer reads stage s
  }
  return true;
}

// The order of torch.argmax: NaN above every number (the first NaN wins), otherwise the larger value, and between
// equal values (-0.0 == +0.0) the lower column.  A strict total order on (value, column), so any combination order
// gives the same winner.
__device__ __forceinline__ bool argmax_before(float v, int col, float best, int best_col) {
  const bool v_nan = v != v, best_nan = best != best;
  if (v_nan || best_nan) return v_nan && (!best_nan || col < best_col);
  return v > best || (v == best && col < best_col);
}

// Philox4x32-10 (Random123; the round of curand_philox4x32_x.h): the four words of counter c under key k.
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

// Gumbel noise of one random word: u = (2·(x >> 9) + 1)·2^-24 is exact and strictly inside (0, 1), g = -log(-log u).
__device__ __forceinline__ float gumbel_of(uint32_t x) {
  const float u = (float)(2u * (x >> 9) + 1u) * 5.9604644775390625e-8f;
  return -logf(-logf(u));
}

// One column pair (col, col + 1) of a layer in rows r and r + 8: y0 = act(a0 + bias, a1 + bias) of row r, y1 of row
// r + 8, each rounded once to bf16.  A column >= n_valid gets no bias.
__device__ __forceinline__ void layer_pair(float a0, float a1, float a2, float a3, const __nv_bfloat16* bias, int col,
                                           int n_valid, int relu, __nv_bfloat162& y0, __nv_bfloat162& y1) {
  float v[4] = {a0, a1, a2, a3};
  // no add at all without a bias: -0.0 accumulators stay -0.0 (adding 0 would make them +0.0).  (The bias is read
  // here rather than before the main loop: 64 more live registers would make the 256-wide instantiation spill.)
  if (bias != nullptr) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      if (col + c < n_valid) {
        const float b = __bfloat162float(bias[col + c]);
        v[c] += b;
        v[2 + c] += b;
      }
    }
  }
  if (relu) {
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = fmaxf(v[q], 0.f);
  }
  y0 = __floats2bfloat162_rn(v[0], v[1]);
  y1 = __floats2bfloat162_rn(v[2], v[3]);
}

// The sampling epilogue of a head tile (mlp_layer_wgmma_kernel with log_probs): rows r = row and row + 8 of the
// thread, global rows row_base + r.  A loop of its own, so that the greedy loop keeps its compact code.  Pass 1 rounds
// the logits once and keeps them as bf16 pairs (half the registers of the fp32 accumulators it frees: the 256-wide
// instantiation would spill holding the accumulators, or the bias, through pass 2) and takes each row's largest logit
// m across the quad (NaN skipped: it reaches the sum instead); pass 2 draws one Philox call per column pair < n_valid
// and row, ranks fp32(logit + noise) in torch.argmax order and sums exp(logit - m) without a running rescale.  A logit equal to m adds 1 without an exp, so an all -inf (or a +inf) maximum never forms
// exp(inf - inf): such rows end with a NaN log-probability, as in torch, and -inf logits beside a finite m add 0.
template <int BLOCK_N>
__device__ __forceinline__ void sample_epilogue(const float (&acc)[BLOCK_N / 2], const __nv_bfloat16* bias, int col0,
                                                int n_valid, int relu, int row, bool st0, bool st1, int64_t* actions,
                                                float* log_probs, uint64_t seed, uint64_t row_base) {
  float mx[2] = {-INFINITY, -INFINITY};
  __nv_bfloat162 y[BLOCK_N / 4];   // y[2j + h]: columns (col, col + 1) of row + 8h
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= n_valid) continue;
    layer_pair(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col, n_valid, relu, y[2 * j],
               y[2 * j + 1]);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float v = q & 1 ? __high2float(y[2 * j + (q >> 1)]) : __low2float(y[2 * j + (q >> 1)]);
      if (col + (q & 1) < n_valid && v > mx[q >> 1]) mx[q >> 1] = v;
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      const float o = __shfl_xor_sync(0xffffffffu, mx[h], m);
      if (o > mx[h]) mx[h] = o;
    }
  }
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  float best[2] = {-INFINITY, -INFINITY}, best_y[2] = {0.f, 0.f}, sum[2] = {0.f, 0.f};
  int best_col[2] = {INT_MAX, INT_MAX};
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= n_valid) continue;   // a pair wholly past the head draws no noise
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint64_t i = row_base + (uint64_t)(row + 8 * h);
      const uint4 x = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)col >> 1, 0u), key);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (col + c >= n_valid) continue;
        const float v = c ? __high2float(y[2 * j + h]) : __low2float(y[2 * j + h]);
        const float s = v + gumbel_of(c ? x.y : x.x);
        if (argmax_before(s, col + c, best[h], best_col[h])) {
          best[h] = s;
          best_col[h] = col + c;
          best_y[h] = v;
        }
        sum[h] += v == mx[h] ? 1.f : expf(v - mx[h]);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best[h], m);
      const int oc = __shfl_xor_sync(0xffffffffu, best_col[h], m);
      const float oy = __shfl_xor_sync(0xffffffffu, best_y[h], m);
      sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], m);
      if (argmax_before(ov, oc, best[h], best_col[h])) {
        best[h] = ov;
        best_col[h] = oc;
        best_y[h] = oy;
      }
    }
  }
  if ((threadIdx.x & 3) == 0) {
    if (st0) {
      actions[row] = best_col[0];
      log_probs[row] = best_y[0] - mx[0] - logf(sum[0]);
    }
    if (st1) {
      actions[row + 8] = best_col[1];
      log_probs[row + 8] = best_y[1] - mx[1] - logf(sum[1]);
    }
  }
}

// The Gaussian epilogue of a head tile (mlp_layer_wgmma_kernel with log_std): rows r = row and row + 8 of the thread,
// global rows row_base + r.  A compact loop of its own, apart from the greedy loop and sample_epilogue: fully unrolled
// here (as those are) it made the kernel half as large again, and ptxas then scheduled sample_epilogue differently and
// 3-9 % slower.  So the unrolled part only rounds the logits once (layer_pair: μ, the value ktb_mlp_bf16_policy
// stores) and parks them as bf16 pairs in the TMA ring, each warp in the 16 A rows of every stage that only its own
// accumulator rows are made of: once the warp's wgmmas are waited for nothing reads or writes them again (every load
// has landed, and no other warp's wgmma reads those rows).  A rolled loop then makes one pass over the column pairs
// < n_valid: one Philox call per pair and row (counter word 3 = 1: never the Gumbel stream's uniforms),
// z = Φ⁻¹(u) (normcdfinvf, no fast-math; u is never 0.5, so z != 0), the action μ + σ·z rounded twice (no FMA
// contraction), stored as float2 where the row stride and the base allow and as scalars otherwise, and
// Σ (0.5·z² + log_std) per row for the log-probability, which does not read μ.
template <int BLOCK_N, int STAGES>
__device__ __forceinline__ void gaussian_epilogue(const float (&acc)[BLOCK_N / 2], const __nv_bfloat16* bias, int col0,
                                                  int n_valid, int relu, int row, bool st0, bool st1,
                                                  const float* log_std, float* actions, float* log_probs,
                                                  uint64_t seed, uint64_t row_base) {
  // opaque copies of the inputs this epilogue shares with the others: without them the compiler hoists the common
  // index and address arithmetic above the mode branch, and ptxas schedules sample_epilogue 2-3 % slower
  asm volatile("" : "+l"(seed), "+l"(row_base), "+l"(bias), "+r"(col0), "+r"(n_valid), "+r"(row));
  using S = MlpSmem<BLOCK_N, STAGES>;
  static_assert(BLOCK_N / 64 <= STAGES, "each warp's bf16 pairs fill its 16 A rows of BLOCK_N / 64 stages");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // pair w (= 2j + h) of a lane: stage w / 16, A rows 16·warp .. 16·warp + 15 (2 KiB), word (w % 16)·32 + lane
  uint8_t* mine = smem + (threadIdx.x >> 5) * 16 * 128 + (threadIdx.x & 31) * 4;
  auto slot = [&](int w) { return reinterpret_cast<__nv_bfloat162*>(mine + (w >> 4) * S::kStageBytes + (w & 15) * 128); };
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= n_valid) continue;
    layer_pair(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col, n_valid, relu, *slot(2 * j),
               *slot(2 * j + 1));
  }
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const bool pairs = (n_valid & 1) == 0 && ((uintptr_t)actions & 7) == 0;
  float sum[2] = {0.f, 0.f};
#pragma unroll 1
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= n_valid) break;   // a pair wholly past the head draws no noise
    const __nv_bfloat162 y[2] = {*slot(2 * j), *slot(2 * j + 1)};
    const bool has1 = col + 1 < n_valid;
    const float ls[2] = {log_std[col], has1 ? log_std[col + 1] : 0.f};
    const float sg[2] = {expf(ls[0]), expf(ls[1])};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint64_t i = row_base + (uint64_t)(row + 8 * h);
      const uint4 x = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)col >> 1, 1u), key);
      float a[2];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float u = (float)(2u * ((c ? x.y : x.x) >> 9) + 1u) * 5.9604644775390625e-8f;
        const float z = normcdfinvf(u);
        a[c] = __fadd_rn(c ? __high2float(y[h]) : __low2float(y[h]), __fmul_rn(sg[c], z));
        if (c == 0 || has1) sum[h] += 0.5f * z * z + ls[c];
      }
      if (!(h ? st1 : st0)) continue;
      float* p = actions + (size_t)(row + 8 * h) * n_valid + col;
      if (pairs) {
        *reinterpret_cast<float2*>(p) = make_float2(a[0], a[1]);
      } else {
        p[0] = a[0];
        if (has1) p[1] = a[1];
      }
    }
  }
  // the 4 lanes of a quad hold the columns of the same two rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], m);
  }
  if ((threadIdx.x & 3) == 0) {
    const float c = (float)n_valid * 0.918938533204672742f;   // d_out·0.5·log(2π)
    if (st0) log_probs[row] = -sum[0] - c;
    if (st1) log_probs[row + 8] = -sum[1] - c;
  }
}

// One MLP layer: C[:, col] = act(A · Bᵀ + bias[col]) for col < n_valid, with the bias added to the fp32
// accumulator and the sum rounded once to bf16 (nn.Linear / F.linear), and actions[row] = the argmax of the row's
// ROUNDED values.  One output tile per CTA; blockIdx.x walks N, so the CTAs of one 128-row block run side by side and
// read their A tile from L2 once.  Only rows < rows (A's row count) are stored.  Bias, ReLU and both outputs are
// runtime choices (bias, C and actions may each be null), so one instantiation per tile width serves every layer:
// 256 for the hidden layers, and for the head the smallest of 64 / 128 / 256 that holds d_out = n_valid, so that one
// CTA owns whole rows (gridDim.x == 1, required with actions) and the argmax never leaves it.  Columns >= n_valid
// hold TMA zero fill: they are never stored and never an action.
// With log_probs (and actions; C is then null) the head SAMPLES instead (Gumbel-max): the action of global row
// i = row_base + row is the argmax of fp32(logit_j + g_j) with g_j the Gumbel noise of Philox word j & 1 of counter
// (i, j >> 1) under `seed` (include/ktb200.h), and log_probs[row] = log_softmax(logits)[action] in fp32.
// With log_std (and gauss_actions and log_probs; C and actions are then null) the head draws Gaussian actions
// instead: gauss_actions[row, j] = logit_j + exp(log_std_j)·z_j with z_j = Φ⁻¹(u) of Philox word j & 1 of counter
// (i, j >> 1, 1), and log_probs[row] the diagonal Normal's log-density of that action (include/ktb200.h).
template <int BLOCK_N, int STAGES>
__global__ void __launch_bounds__(kMlpThreads, 1)
    mlp_layer_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                           const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ C,
                           int64_t* __restrict__ actions, float* __restrict__ log_probs, uint64_t seed,
                           uint64_t row_base, const float* __restrict__ log_std, float* __restrict__ gauss_actions,
                           int ldc, int n_valid, int K, int rows, int relu) {
  const int n0 = blockIdx.x * BLOCK_N;
  const int m0 = blockIdx.y * kMlpBlockM;
  const int lane = threadIdx.x & 31;
  const int col0 = n0 + 2 * (lane & 3);
  float acc[BLOCK_N / 2];
  if (!mlp_tile_mainloop<BLOCK_N, STAGES>(&map_a, &map_b, K, m0, n0, acc)) return;
  const int warp = threadIdx.x >> 5;
  const int wg = warp >> 2;

  // accumulator layout of m64nNk16: acc[4j + 2h + c] is row 16*(warp%4) + lane/4 + 8h, column 8j + 2*(lane%4) + c
  const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const bool st0 = row < rows, st1 = row + 8 < rows;
  if (log_std != nullptr) {
    gaussian_epilogue<BLOCK_N, STAGES>(acc, bias, col0, n_valid, relu, row, st0, st1, log_std, gauss_actions,
                                       log_probs, seed, row_base);
    return;
  }
  if (log_probs != nullptr) {
    sample_epilogue<BLOCK_N>(acc, bias, col0, n_valid, relu, row, st0, st1, actions, log_probs, seed, row_base);
    return;
  }
  // a column pair is one 4-byte store where the base and an even row stride allow it; rows of an odd d_out are
  // only 2-byte aligned and take scalar stores
  const bool pairs = C != nullptr && (ldc & 1) == 0 && ((uintptr_t)C & 3) == 0;
  if (pairs && actions == nullptr && n0 + BLOCK_N <= n_valid) {
    // every column of the tile is stored, in pairs, and no action is taken (every hidden-layer tile): the loop below
    // without its per-column masks and branches
    __nv_bfloat16* p0 = C + (size_t)row * ldc + col0;
    __nv_bfloat16* p1 = p0 + (size_t)8 * ldc;
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      __nv_bfloat162 y0, y1;
      layer_pair(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col0 + 8 * j, n_valid, relu, y0, y1);
      if (st0) *reinterpret_cast<__nv_bfloat162*>(p0 + 8 * j) = y0;
      if (st1) *reinterpret_cast<__nv_bfloat162*>(p1 + 8 * j) = y1;
    }
    return;
  }
  float best[2] = {-INFINITY, -INFINITY};
  int best_col[2] = {INT_MAX, INT_MAX};
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    __nv_bfloat162 y0, y1;
    layer_pair(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col, n_valid, relu, y0, y1);
    if (C != nullptr) {
      __nv_bfloat16* p0 = C + (size_t)row * ldc + col;
      __nv_bfloat16* p1 = p0 + (size_t)8 * ldc;
      if (pairs && col + 1 < n_valid) {
        if (st0) *reinterpret_cast<__nv_bfloat162*>(p0) = y0;
        if (st1) *reinterpret_cast<__nv_bfloat162*>(p1) = y1;
      } else {
        if (st0 && col < n_valid) p0[0] = y0.x;
        if (st1 && col < n_valid) p1[0] = y1.x;
        if (st0 && col + 1 < n_valid) p0[1] = y0.y;
        if (st1 && col + 1 < n_valid) p1[1] = y1.y;
      }
    }
    if (actions != nullptr) {
      const float r[4] = {__low2float(y0), __high2float(y0), __low2float(y1), __high2float(y1)};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int h = q >> 1, c = col + (q & 1);
        if (c < n_valid && argmax_before(r[q], c, best[h], best_col[h])) {
          best[h] = r[q];
          best_col[h] = c;
        }
      }
    }
  }
  if (actions != nullptr) {
    // the 4 lanes of a quad hold the columns of the same two rows
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int m = 1; m <= 2; m <<= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best[h], m);
        const int oc = __shfl_xor_sync(0xffffffffu, best_col[h], m);
        if (argmax_before(ov, oc, best[h], best_col[h])) {
          best[h] = ov;
          best_col[h] = oc;
        }
      }
    }
    if ((lane & 3) == 0) {
      if (st0) actions[row] = best_col[0];
      if (st1) actions[row + 8] = best_col[1];
    }
  }
}

// ---- host side --------------------------------------------------------------------------------------
typedef CUresult (*PFN_tensorMapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                             const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                             CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                             CUtensorMapFloatOOBfill);
static PFN_tensorMapEncodeTiled g_encode = nullptr;
static std::once_flag g_encode_once;

static int get_encoder() {
  std::call_once(g_encode_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      g_encode = reinterpret_cast<PFN_tensorMapEncodeTiled>(fn);
  });
  KTB_REQUIRE(g_encode != nullptr, KTB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  return KTB_OK;
}

// Row-major bf16 [rows, cols] matrix, box = [box_rows, 64 cols], 128-byte swizzle.
static int encode_map(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows);

// The descriptor depends only on (base, rows, cols, box_rows): weights, scratch and staging repeat every chunk and
// every call, so each host thread keeps a small cache (the per-rank issue loop is host-bound at 8 GPUs).
static int make_map(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  struct Key {
    const void* base;
    uint64_t rows, cols;
    uint32_t box;
    bool operator==(const Key& o) const { return base == o.base && rows == o.rows && cols == o.cols && box == o.box; }
  };
  struct Slot {
    Key key;
    CUtensorMap map;
    bool used = false;
  };
  constexpr int kSlots = 64;
  thread_local Slot cache[kSlots];
  const Key k{base, rows, cols, box_rows};
  const size_t h = ((uintptr_t)base >> 8) * 0x9E3779B97F4A7C15ull + rows * 31 + cols * 7 + box_rows;
  Slot& s = cache[h % kSlots];
  if (s.used && s.key == k) {
    *map = s.map;
    return KTB_OK;
  }
  int rc = encode_map(map, base, rows, cols, box_rows);
  if (rc) return rc;
  s.key = k;
  s.map = *map;
  s.used = true;
  return KTB_OK;
}

static int encode_map(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)kMlpBlockK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  KTB_REQUIRE(r == CUDA_SUCCESS, KTB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return KTB_OK;
}

// cudaFuncSetAttribute once per (kernel, device) instead of on every launch.
template <typename KernelT>
static int ensure_smem_attr(KernelT kfn, int smem_bytes, std::atomic<unsigned>& done_mask, int dev) {
  if (dev >= 0 && dev < 32 && (done_mask.load(std::memory_order_acquire) & (1u << dev))) return KTB_OK;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(max dynamic shared memory = %d) failed: %s", smem_bytes, cudaGetErrorString(e));
    return KTB_ERR_CUDA;
  }
  if (dev >= 0 && dev < 32) done_mask.fetch_or(1u << dev, std::memory_order_release);
  return KTB_OK;
}

// What a policy head computes; each entry point names its own.
enum class HeadKind {
  kGreedy,     // bf16 logits and/or int64 argmax actions
  kSample,     // Gumbel-max int64 actions and fp32 log_probs
  kGaussian,   // fp32 actions [rows, d_out] (gauss_actions) drawn with log_std, and fp32 log_probs
};

// The outputs of a head launch; a hidden layer's launch passes an empty one.  Pointers the head kind does not store
// are null.  Row r of the launch draws the noise of global row row_base + r.
struct HeadOut {
  void* logits = nullptr;
  int64_t* actions = nullptr;
  float* log_probs = nullptr;
  uint64_t seed = 0, row_base = 0;
  const float* log_std = nullptr;
  float* gauss_actions = nullptr;

  // The same outputs from row r0 of the call on.
  HeadOut from_row(size_t r0, int d_out) const {
    HeadOut h = *this;
    if (logits) h.logits = static_cast<__nv_bfloat16*>(logits) + r0 * d_out;
    if (actions) h.actions += r0;
    if (log_probs) h.log_probs += r0;
    if (gauss_actions) h.gauss_actions += r0 * d_out;
    h.row_base += r0;
    return h;
  }
};

template <int BLOCK_N>
static int launch_layer(int dev, const void* A, const void* B, const void* bias, void* C, const HeadOut& head,
                        size_t M, int N, int K, int ldc, bool relu, cudaStream_t stream) {
  using S = MlpSmem<BLOCK_N, kMlpStages>;
  static_assert(S::kTotal <= 232448, "the TMA ring must fit the 227 KiB a block may own");
  CUtensorMap ma, mb;
  int rc = make_map(&ma, A, M, (uint64_t)K, kMlpBlockM);
  if (rc) return rc;
  rc = make_map(&mb, B, (uint64_t)N, (uint64_t)K, BLOCK_N);
  if (rc) return rc;
  auto kfn = mlp_layer_wgmma_kernel<BLOCK_N, kMlpStages>;
  static std::atomic<unsigned> attr_done{0};
  rc = ensure_smem_attr(kfn, S::kTotal, attr_done, dev);
  if (rc) return rc;
  dim3 grid((unsigned)((N + BLOCK_N - 1) / BLOCK_N), (unsigned)((M + kMlpBlockM - 1) / kMlpBlockM));
  kfn<<<grid, kMlpThreads, S::kTotal, stream>>>(ma, mb, static_cast<const __nv_bfloat16*>(bias),
                                                static_cast<__nv_bfloat16*>(C), head.actions, head.log_probs,
                                                head.seed, head.row_base, head.log_std, head.gauss_actions, ldc, N, K,
                                                (int)M, relu);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

// Weights and biases (each bias may be null) of one MLP call, and its head.
struct MlpParams {
  const void *W1, *b1, *W2, *b2, *W3, *b3;
  HeadKind kind;
  HeadOut out;
};

// Rows [r0, r0 + rows) of a call: the hidden layers h1 = relu(a1 · W1ᵀ (+ b1)) and h2 = relu(h1 · W2ᵀ (+ b2)), then
// the head from h2 in the smallest tile that holds d_out.  `consumed`, unless null, is recorded once layer 1 has read
// a1.
static int mlp_chunk(int dev, const MlpParams& p, const void* a1, void* h1, void* h2, size_t r0, size_t rows, int d_in,
                     int d_hidden, int d_out, cudaEvent_t consumed, cudaStream_t st) {
  int rc = launch_layer<256>(dev, a1, p.W1, p.b1, h1, HeadOut{}, rows, d_hidden, d_in, d_hidden, true, st);
  if (rc) return rc;
  if (consumed) KTB_CK(cudaEventRecord(consumed, st));
  rc = launch_layer<256>(dev, h1, p.W2, p.b2, h2, HeadOut{}, rows, d_hidden, d_hidden, d_hidden, true, st);
  if (rc) return rc;
  const HeadOut h = p.out.from_row(r0, d_out);
  const auto head = d_out <= 64 ? launch_layer<64> : d_out <= 128 ? launch_layer<128> : launch_layer<256>;
  return head(dev, h2, p.W3, p.b3, h.logits, h, rows, d_out, d_hidden, d_out, false, st);
}

// The checks every MLP entry shares: the layer widths the tiles divide, the head (the outputs its kind stores, width,
// element-aligned pointers; skipped for an empty call, which stores nothing and may pass null outputs) and the
// 16-byte alignment TMA needs of every matrix it loads (`obs` is the first layer's input).
static int mlp_check(const char* fn, size_t M, int d_in, int d_hidden, int d_out, const MlpParams& p, const void* obs,
                     const void* scratch, const void* stage) {
  KTB_REQUIRE(d_in > 0 && d_in % kMlpBlockK == 0, KTB_ERR_ARG, "%s: d_in=%d must be a multiple of 64", fn, d_in);
  KTB_REQUIRE(d_hidden > 0 && d_hidden % 256 == 0, KTB_ERR_ARG, "%s: d_hidden=%d must be a multiple of 256", fn,
              d_hidden);
  if (M > 0) {
    const HeadOut& o = p.out;
    switch (p.kind) {
      case HeadKind::kGreedy:
        KTB_REQUIRE(o.logits || o.actions, KTB_ERR_ARG, "%s: logits and actions are both null", fn);
        break;
      case HeadKind::kSample:
        KTB_REQUIRE(o.actions && o.log_probs, KTB_ERR_ARG, "%s: actions and log_probs are required", fn);
        break;
      case HeadKind::kGaussian:
        KTB_REQUIRE(o.log_std && o.gauss_actions && o.log_probs, KTB_ERR_ARG,
                    "%s: log_std, actions and log_probs are required", fn);
        KTB_REQUIRE((((uintptr_t)o.log_std | (uintptr_t)o.gauss_actions) & 3) == 0, KTB_ERR_ARG,
                    "%s: log_std and actions must be 4-byte aligned", fn);
        break;
    }
    KTB_REQUIRE(d_out >= 1, KTB_ERR_ARG, "%s: d_out=%d must be positive", fn, d_out);
    KTB_REQUIRE(d_out <= 256, KTB_ERR_UNSUPPORTED, "%s: d_out=%d (heads up to 256 wide)", fn, d_out);
    // outputs the kind does not store are null and pass
    KTB_REQUIRE((((uintptr_t)o.logits | (uintptr_t)p.b1 | (uintptr_t)p.b2 | (uintptr_t)p.b3) & 1) == 0, KTB_ERR_ARG,
                "%s: logits and biases must be 2-byte aligned", fn);
    KTB_REQUIRE(((uintptr_t)o.actions & 7) == 0, KTB_ERR_ARG, "%s: actions must be 8-byte aligned", fn);
    KTB_REQUIRE(((uintptr_t)o.log_probs & 3) == 0, KTB_ERR_ARG, "%s: log_probs must be 4-byte aligned", fn);
  }
  KTB_REQUIRE((((uintptr_t)obs | (uintptr_t)p.W1 | (uintptr_t)p.W2 | (uintptr_t)p.W3 | (uintptr_t)scratch |
                (uintptr_t)stage) & 15) == 0,
              KTB_ERR_ARG, "%s: obs, weights, scratch and stage must be 16-byte aligned", fn);
  return KTB_OK;
}
}  // namespace ktb

using namespace ktb;

extern "C" {

size_t ktb_mlp_scratch_bytes(size_t M, int d_hidden) {
  const size_t rows = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  return 2 * rows * (size_t)d_hidden * 2;
}

size_t ktb_mlp_stage_bytes(size_t M, int d_in) {
  const size_t rows = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  return 2 * rows * (size_t)d_in * 2;
}

// ktb_set_tuning(22, v): staged pulls by a pull kernel (0, default) or by copy engine (1)
int g_mlp_stage_ce = 0;

static int mlp_run(const char* fn, int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                   const MlpParams& p, void* scratch, void* stage, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  if (M == 0) return KTB_OK;
  KTB_REQUIRE(obs && p.W1 && p.W2 && p.W3 && scratch, KTB_ERR_ARG, "%s: null argument", fn);
  rc = mlp_check(fn, M, d_in, d_hidden, d_out, p, obs, scratch, stage);
  if (rc) return rc;
  KTB_REQUIRE(g_mlp_chunk_rows % kMlpBlockM == 0 && g_mlp_chunk_rows > 0, KTB_ERR_ARG, "%s: bad chunk rows", fn);
  rc = get_encoder();
  if (rc) return rc;
  KTB_GUARD(dev);
  DeviceInfo* di = device_info(dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cudaStream_t side = di->stream_exec;   // pulls the next chunk while this one computes
  const size_t chunk = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  __nv_bfloat16* h1 = static_cast<__nv_bfloat16*>(scratch);
  __nv_bfloat16* h2 = h1 + chunk * (size_t)d_hidden;
  const __nv_bfloat16* x = static_cast<const __nv_bfloat16*>(obs);
  __nv_bfloat16* stg = static_cast<__nv_bfloat16*>(stage);
  const MapParams ident = make_params(1, 0);
  // per-call events: [0] start, [1..2] staged chunk landed (by buffer), [3..4] staging buffer consumed
  cudaEvent_t evs[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  struct EvGuard {
    cudaEvent_t* e;
    ~EvGuard() {
      for (int i = 0; i < 5; ++i)
        if (e[i]) cudaEventDestroy(e[i]);
    }
  } ev_guard{evs};
  static std::mutex side_mu[kMaxDevices];   // the side stream of a device carries one staged call at a time
  std::unique_lock<std::mutex> side_lock;
  if (stg) {
    side_lock = std::unique_lock<std::mutex>(side_mu[dev]);
    for (int i = 0; i < 5; ++i) KTB_CK(cudaEventCreateWithFlags(&evs[i], cudaEventDisableTiming));
    KTB_CK(cudaEventRecord(evs[0], st));            // obs is ready once prior work on `st` is done
    KTB_CK(cudaStreamWaitEvent(side, evs[0], 0));
  }
  size_t c = 0;
  for (size_t r0 = 0; r0 < M; r0 += chunk, ++c) {
    const size_t rows = std::min(chunk, M - r0);
    const __nv_bfloat16* a1 = x + r0 * d_in;
    if (stg) {
      // staged pull: rows of this chunk travel peer → local ONCE (the layer-1 GEMM would otherwise fetch every
      // A tile d_hidden/256 times over NVLink, peer reads being uncached in the local L2)
      const int b = (int)(c & 1);
      __nv_bfloat16* dstb = stg + (size_t)b * chunk * d_in;
      if (c >= 2) KTB_CK(cudaStreamWaitEvent(side, evs[3 + b], 0));   // GEMM 1 of chunk c-2 consumed it
      if (g_mlp_stage_ce) {
        // copy engine pull: no SM of this rank moves observation rows
        KTB_CK(cudaMemcpyAsync(dstb, a1, rows * (size_t)d_in * 2, cudaMemcpyDefault, side));
      } else {
        rc = launch_map(dev, KTB_OP_IDENTITY, KTB_U8, a1, dstb, rows * (size_t)d_in * 2, ident, KTB_VARIANT_AUTO, side);
        if (rc) return rc;
      }
      KTB_CK(cudaEventRecord(evs[1 + b], side));
      KTB_CK(cudaStreamWaitEvent(st, evs[1 + b], 0));
      a1 = dstb;
    }
    // evs[3..4] are null unless staged
    rc = mlp_chunk(dev, p, a1, h1, h2, r0, rows, d_in, d_hidden, d_out, evs[3 + (int)(c & 1)], st);
    if (rc) return rc;
  }
  return KTB_OK;
}

// ---- pushed form: the root PUSHES this rank's observation rows chunk by chunk (ktb_push_scatter_chunked) ------------
namespace ktb {
// Stream-ordered "chunk c has landed": one warp spins on the local ready flag (a timeout raises the sticky status).
__global__ void mlp_wait_ready_kernel(const unsigned long long* ready, unsigned long long seq, unsigned int* status) {
  if (threadIdx.x == 0) (void)spin_until(ready, seq, status);
}
// Stream-ordered completion of the rank's call: everything before it on the stream (incl. the peer-stored logits)
// is visible system-wide before the root sees ack[rank] = seq.
__global__ void mlp_ack_kernel(unsigned long long* ack, unsigned long long seq) {
  if (threadIdx.x == 0) {
    __threadfence_system();
    st_release_sys(ack, seq);
  }
}
}  // namespace ktb

static int mlp_pushed_run(const char* fn, int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                          int d_hidden, int d_out, const MlpParams& p, void* scratch, void* ctrl_local,
                          void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(stage_local && ctrl_local && ctrl_root_peer && p.W1 && p.W2 && p.W3 && scratch, KTB_ERR_ARG,
              "%s: null argument", fn);
  KTB_REQUIRE(rank >= 0 && rank < 16 && seq > 0, KTB_ERR_ARG, "%s: bad rank/seq", fn);
  KTB_REQUIRE(M % kMlpBlockM == 0, KTB_ERR_ARG, "%s: M=%zu must be a multiple of %d", fn, M, kMlpBlockM);
  KTB_REQUIRE(chunk_rows > 0 && chunk_rows % kMlpBlockM == 0, KTB_ERR_ARG,
              "%s: chunk_rows=%zu must be a positive multiple of %d", fn, chunk_rows, kMlpBlockM);
  rc = mlp_check(fn, M, d_in, d_hidden, d_out, p, stage_local, scratch, nullptr);
  if (rc) return rc;
  const size_t n_chunks = (M + chunk_rows - 1) / chunk_rows;
  KTB_REQUIRE(n_chunks <= KTB_PUSH_MAX_CHUNKS, KTB_ERR_ARG, "%s: %zu chunks exceed %d", fn, n_chunks,
              KTB_PUSH_MAX_CHUNKS);
  KTB_REQUIRE(M * (size_t)d_in * 2 <= stage_stride, KTB_ERR_ARG, "%s: shard exceeds stage_stride", fn);
  rc = get_encoder();
  if (rc) return rc;
  KTB_GUARD(dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* cl = static_cast<uint8_t*>(ctrl_local);
  const unsigned long long* ready = reinterpret_cast<const unsigned long long*>(cl + KTB_CTRL_READY);
  unsigned int* status = reinterpret_cast<unsigned int*>(cl + KTB_CTRL_STATUS);
  unsigned long long* ack =
      reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ctrl_root_peer) + KTB_CTRL_ACK) + rank;
  const __nv_bfloat16* x =
      reinterpret_cast<const __nv_bfloat16*>(static_cast<const uint8_t*>(stage_local) + (size_t)(seq & 1) * stage_stride);
  __nv_bfloat16* h1 = static_cast<__nv_bfloat16*>(scratch);
  __nv_bfloat16* h2 = h1 + std::min(chunk_rows, M) * (size_t)d_hidden;
  size_t c = 0;
  for (size_t r0 = 0; r0 < M; r0 += chunk_rows, ++c) {
    const size_t rows = std::min(chunk_rows, M - r0);
    mlp_wait_ready_kernel<<<1, 32, 0, st>>>(ready + c, seq, status);
    KTB_CK(cudaGetLastError());
    rc = mlp_chunk(dev, p, x + r0 * d_in, h1, h2, r0, rows, d_in, d_hidden, d_out, nullptr, st);
    if (rc) return rc;
  }
  mlp_ack_kernel<<<1, 32, 0, st>>>(ack, seq);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

// ktb_mlp_bf16, _staged and _pushed are the policy form without biases, with a 64-wide head and logits only.  Each
// checks that narrower contract (after the device, and for the pull forms after an empty call, which returns first)
// and then runs the policy form.
int ktb_mlp_bf16_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_out,
                        const void* W1, const void* W2, const void* W3, void* logits, void* scratch, void* ctrl_local,
                        void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const char* fn = "ktb_mlp_bf16_pushed";
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(logits || M == 0, KTB_ERR_ARG, "%s: null argument", fn);
  KTB_REQUIRE(d_out == 64, KTB_ERR_UNSUPPORTED, "%s: d_out=%d (the 64-wide head)", fn, d_out);
  const MlpParams p{W1, nullptr, W2, nullptr, W3, nullptr, HeadKind::kGreedy, {logits}};
  return mlp_pushed_run(fn, dev, stage_local, stage_stride, M, d_in, d_hidden, d_out, p, scratch, ctrl_local,
                        ctrl_root_peer, rank, chunk_rows, seq, stream);
}

int ktb_mlp_bf16_policy_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden,
                               int d_out, const void* W1, const void* b1, const void* W2, const void* b2,
                               const void* W3, const void* b3, void* logits, int64_t* actions, void* scratch,
                               void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                               unsigned long long seq, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGreedy, {logits, actions}};
  return mlp_pushed_run("ktb_mlp_bf16_policy_pushed", dev, stage_local, stage_stride, M, d_in, d_hidden, d_out, p,
                        scratch, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq, stream);
}

static int mlp_run_64(const char* fn, int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                      const void* W1, const void* W2, const void* W3, void* logits, void* scratch, void* stage,
                      uintptr_t stream) {
  int rc = require_device(dev);
  if (rc || M == 0) return rc;
  KTB_REQUIRE(logits, KTB_ERR_ARG, "%s: null argument", fn);
  KTB_REQUIRE(d_out == 64, KTB_ERR_UNSUPPORTED, "%s: d_out=%d (the 64-wide head)", fn, d_out);
  KTB_REQUIRE(((uintptr_t)logits & 15) == 0, KTB_ERR_ARG, "%s: logits must be 16-byte aligned", fn);
  const MlpParams p{W1, nullptr, W2, nullptr, W3, nullptr, HeadKind::kGreedy, {logits}};
  return mlp_run(fn, dev, obs, M, d_in, d_hidden, d_out, p, scratch, stage, stream);
}

int ktb_mlp_bf16(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                 const void* W2, const void* W3, void* logits, void* scratch, uintptr_t stream) {
  return mlp_run_64("ktb_mlp_bf16", dev, obs, M, d_in, d_hidden, d_out, W1, W2, W3, logits, scratch, nullptr, stream);
}

int ktb_mlp_bf16_staged(int dev, const void* obs_peer, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                        const void* W2, const void* W3, void* logits, void* scratch, void* stage, uintptr_t stream) {
  KTB_REQUIRE(stage, KTB_ERR_ARG, "ktb_mlp_bf16_staged: null stage buffer");
  return mlp_run_64("ktb_mlp_bf16_staged", dev, obs_peer, M, d_in, d_hidden, d_out, W1, W2, W3, logits, scratch, stage,
                    stream);
}

int ktb_mlp_bf16_policy(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                        const void* b1, const void* W2, const void* b2, const void* W3, const void* b3, void* logits,
                        int64_t* actions, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGreedy, {logits, actions}};
  return mlp_run("ktb_mlp_bf16_policy", dev, obs, M, d_in, d_hidden, d_out, p, scratch, stage, stream);
}

int ktb_mlp_bf16_policy_sample(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                               const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                               uint64_t seed, uint64_t row_base, int64_t* actions, float* log_probs, void* scratch,
                               void* stage, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}};
  return mlp_run("ktb_mlp_bf16_policy_sample", dev, obs, M, d_in, d_hidden, d_out, p, scratch, stage, stream);
}

int ktb_mlp_bf16_policy_sample_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                      int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                      const void* b2, const void* W3, const void* b3, uint64_t seed, uint64_t row_base,
                                      int64_t* actions, float* log_probs, void* scratch, void* ctrl_local,
                                      void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq,
                                      uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}};
  return mlp_pushed_run("ktb_mlp_bf16_policy_sample_pushed", dev, stage_local, stage_stride, M, d_in, d_hidden, d_out,
                        p, scratch, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq, stream);
}

int ktb_mlp_bf16_policy_gaussian(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                 const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                                 const float* log_std, uint64_t seed, uint64_t row_base, float* actions,
                                 float* log_probs, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGaussian,
                    {nullptr, nullptr, log_probs, seed, row_base, log_std, actions}};
  return mlp_run("ktb_mlp_bf16_policy_gaussian", dev, obs, M, d_in, d_hidden, d_out, p, scratch, stage, stream);
}

int ktb_mlp_bf16_policy_gaussian_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                        int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                        const void* b2, const void* W3, const void* b3, const float* log_std,
                                        uint64_t seed, uint64_t row_base, float* actions, float* log_probs,
                                        void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                        size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGaussian,
                    {nullptr, nullptr, log_probs, seed, row_base, log_std, actions}};
  return mlp_pushed_run("ktb_mlp_bf16_policy_gaussian_pushed", dev, stage_local, stage_stride, M, d_in, d_hidden,
                        d_out, p, scratch, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq, stream);
}

}  // extern "C"

