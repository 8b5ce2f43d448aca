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
//   * an epilogue from the fp32 register accumulators, chosen at compile time by HeadKind: optional
//     bias (nn.Linear) and bf16 rounding, then for the hidden layers ReLU and full-tile stores, and
//     for the head one of: logits masked to its width and/or the greedy action of every row; an
//     action sampled by seeded Gumbel-max with its log-probability (either of these two optionally under a per-row
//     legal-action mask, a runtime input, and either optionally split into groups of columns with one greedy or
//     sampled action per group, a multi-discrete action space); or Gaussian actions with their
//     log-probability (the sampled and Gaussian heads optionally with a critic's state value, one more head column,
//     also a runtime input) — the head's outputs may be peer pointers into the root GPU's result arena,
//     which fuses the gather into the epilogue.
// Warp roles (288 threads): warps 0-7 = two consumer warpgroups, warp 8 = TMA producer (one lane).
// Activations are rounded to bf16 between layers (like the eager torch module); rows are processed
// in chunks whose hidden activations stay resident in the 50 MB L2.  One kernel template
// (mlp_layer_wgmma_kernel<BLOCK_N, STAGES, HeadKind>) runs every layer of every entry point.
// On the host every entry point sits on two axes: its head (MlpParams: weights, biases, HeadKind and outputs) and its
// form (MlpFeed: how each row chunk reaches layer 1 — read in place, pulled from a peer into `stage`, or pushed by the
// root and waited for in-stream).  Each entry only builds the two and calls mlp_run, which checks them, then runs one
// chunk loop over mlp_chunk (layer 1, layer 2, head).
#include "ktb_common.cuh"

#include <cuda.h>
#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <mutex>
#include <type_traits>

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
int g_mlp_stage_ce = 0;        // ktb_set_tuning key 22: staged pulls by a pull kernel (0, default) or by copy engine (1)

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
// the accumulators of those rows and columns are 0 and the epilogue decides what to store.  map_a holds two maps of A:
// the K blocks kb < kb_split come from map_a[0] at column 64·kb, the rest from map_a[1] at column 64·(kb − kb_split),
// so a critic's layer 1 reads the observation rows where they are and its action tile beside them.  Every other layer
// has kb_split = K / 64.
template <int BLOCK_N, int STAGES>
__device__ __forceinline__ bool mlp_tile_mainloop(const CUtensorMap* map_a, const CUtensorMap* map_b, int K,
                                                  int kb_split, int m0, int n0, float (&acc)[BLOCK_N / 2]) {
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
      if (kb_split < num_kb) prefetch_tensormap(map_a + 1);
      prefetch_tensormap(map_b);
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        mbar_wait(&empty[s], ((kb / STAGES) & 1) ^ 1);
        uint8_t* a_dst = smem + (size_t)s * S::kStageBytes;
        mbar_expect_tx(&full[s], S::kStageBytes);
        const bool first = kb < kb_split;
        tma_load_2d(a_dst, map_a + !first, (first ? kb : kb - kb_split) * kMlpBlockK, m0, &full[s]);
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

// Gumbel noise of one random word: u = (2·(x >> 9) + 1)·2^-24 is exact and strictly inside (0, 1), g = -log(-log u).
__device__ __forceinline__ float gumbel_of(uint32_t x) {
  const float u = (float)(2u * (x >> 9) + 1u) * 5.9604644775390625e-8f;
  return -logf(-logf(u));
}

// torch.relu: max.NaN returns NaN when an operand is NaN (fmaxf would return the 0), +inf stays +inf and -inf gives
// +0.0.  Before a bf16 rounding ptxas folds it into the conversion (F2FP.RELU, which keeps NaN), so it costs no
// instruction.  A zero's sign may differ from torch's; a hidden zero's sign never reaches an output.
__device__ __forceinline__ float relu_keep_nan(float v) {
  float r;
  asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(v));
  return r;
}

// One column pair (col, col + 1) of a layer in rows r and r + 8: y0 = act(a0 + bias, a1 + bias) of row r, y1 of row
// r + 8, each rounded once to bf16; act is ReLU (relu_keep_nan: a NaN stays NaN, as in torch) in the hidden layers
// and the identity in the head.  A column >= n_valid gets no bias.
template <bool RELU>
__device__ __forceinline__ void layer_pair(float a0, float a1, float a2, float a3, const __nv_bfloat16* bias, int col,
                                           int n_valid, __nv_bfloat162& y0, __nv_bfloat162& y1) {
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
  if constexpr (RELU) {
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = relu_keep_nan(v[q]);
  }
  y0 = __floats2bfloat162_rn(v[0], v[1]);
  y1 = __floats2bfloat162_rn(v[2], v[3]);
}

// The columns a head epilogue ranks, one bit per column of the thread: bit 2j + c of live[h] is column col0 + 8j + c of
// row + 8h.  Without a mask a column is live when it is < n_valid (a closed form, no loop); with a legal-action mask
// [rows, n_valid] (row-major, nonzero byte: legal) it must also be legal, and the bytes are read in a rolled loop only
// for stored rows (st0, st1) and columns < n_valid, so nothing past legal[rows, n_valid] is touched.  The epilogues skip
// dead columns in the tests they already make for columns past n_valid, which is what ranking and summing
// logits.masked_fill(~legal, -inf) comes to; the masked code stays out of the unrolled loops of the unmasked heads.
template <int BLOCK_N>
using ColBits = typename std::conditional<(BLOCK_N > 128), unsigned long long, unsigned>::type;

template <int BLOCK_N>
__device__ __forceinline__ void live_columns(const uint8_t* mask, int row, int col0, int n_valid, bool st0, bool st1,
                                             ColBits<BLOCK_N> (&live)[2]) {
  using B = ColBits<BLOCK_N>;
  constexpr int kBits = BLOCK_N / 4;
  const int r = n_valid - col0;   // columns col0 + 8j + c < n_valid: 8j < r (even bits), 8j + 1 < r (odd bits)
  const int ne = r <= 0 ? 0 : min((r + 7) / 8, BLOCK_N / 8);
  const int no = r <= 1 ? 0 : min((r + 6) / 8, BLOCK_N / 8);
  const auto low = [](int n) { return n >= kBits ? ~B(0) : (B(1) << n) - B(1); };
  live[0] = live[1] = (B(0x5555555555555555ull) & low(2 * ne)) | (B(0xAAAAAAAAAAAAAAAAull) & low(2 * no));
  if (mask == nullptr) return;
  const uint8_t* m0 = mask + (size_t)row * n_valid + col0;
  const uint8_t* m1 = m0 + (size_t)8 * n_valid;
  B l0 = 0, l1 = 0;
#pragma unroll 1
  for (int k = 0; k < kBits; ++k) {
    if (!((live[0] >> k) & 1)) break;   // columns grow with k: the first column past n_valid ends the row
    const int off = 8 * (k >> 1) + (k & 1);
    if (st0 && m0[off] != 0) l0 |= B(1) << k;
    if (st1 && m1[off] != 0) l1 |= B(1) << k;
  }
  live[0] = l0;
  live[1] = l1;
}

// Every column of a tile stored in pairs, with no per-column masks or branches: the hidden layers (RELU; d_hidden is
// a multiple of 256 and the scratch is 16-byte aligned, so every hidden tile is full and pair-aligned) and a greedy
// head whose one tile is full and pair-aligned and that takes no actions.  C has n_valid columns.
template <int BLOCK_N, bool RELU>
__device__ __forceinline__ void store_tile(const float (&acc)[BLOCK_N / 2], const __nv_bfloat16* bias,
                                           __nv_bfloat16* C, int col0, int n_valid, int row, bool st0, bool st1) {
  __nv_bfloat16* p0 = C + (size_t)row * n_valid + col0;
  __nv_bfloat16* p1 = p0 + (size_t)8 * n_valid;
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    __nv_bfloat162 y0, y1;
    layer_pair<RELU>(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col0 + 8 * j, n_valid, y0, y1);
    if (st0) *reinterpret_cast<__nv_bfloat162*>(p0 + 8 * j) = y0;
    if (st1) *reinterpret_cast<__nv_bfloat162*>(p1 + 8 * j) = y1;
  }
}

// The greedy epilogue of a head tile: logits (C, unless null) masked to the head's n_valid columns over the TMA zero
// fill, and actions[row] (unless null) the argmax of the row's ROUNDED logits.  With a legal-action mask only legal
// columns are ranked (live_columns), a row whose ranked logits are all -inf or that has none takes action 0 as
// torch.argmax does, and a rolled pass overwrites the stored logits of illegal columns with -inf.  The head's one tile
// holds whole rows (n_valid <= BLOCK_N), so the argmax never leaves the CTA.
template <int BLOCK_N>
__device__ __forceinline__ void greedy_epilogue(const float (&acc)[BLOCK_N / 2], const __nv_bfloat16* bias,
                                                __nv_bfloat16* C, int64_t* actions, const uint8_t* mask, int col0,
                                                int n_valid, int row, bool st0, bool st1) {
  // a column pair is one 4-byte store where the base and an even row stride allow it; rows of an odd d_out are
  // only 2-byte aligned and take scalar stores
  const bool pairs = C != nullptr && (n_valid & 1) == 0 && ((uintptr_t)C & 3) == 0;
  if (pairs && actions == nullptr && mask == nullptr && n_valid == BLOCK_N) {
    store_tile<BLOCK_N, false>(acc, bias, C, col0, n_valid, row, st0, st1);
    return;
  }
  ColBits<BLOCK_N> live[2];
  live_columns<BLOCK_N>(mask, row, col0, n_valid, st0, st1, live);
  float best[2] = {-INFINITY, -INFINITY};
  int best_col[2] = {INT_MAX, INT_MAX};
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    __nv_bfloat162 y0, y1;
    layer_pair<false>(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col, n_valid, y0, y1);
    if (C != nullptr) {
      __nv_bfloat16* p0 = C + (size_t)row * n_valid + col;
      __nv_bfloat16* p1 = p0 + (size_t)8 * n_valid;
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
        if (((live[h] >> (2 * j + (q & 1))) & 1) && argmax_before(r[q], c, best[h], best_col[h])) {
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
    if ((threadIdx.x & 3) == 0) {
      if (st0) actions[row] = best[0] == -INFINITY ? 0 : best_col[0];
      if (st1) actions[row + 8] = best[1] == -INFINITY ? 0 : best_col[1];
    }
  }
  if (mask != nullptr && C != nullptr) {
    const __nv_bfloat16 ninf = __ushort_as_bfloat16((unsigned short)0xFF80u);
#pragma unroll 1
    for (int k = 0; k < BLOCK_N / 4; ++k) {
      const int col = col0 + 8 * (k >> 1) + (k & 1);
      if (col >= n_valid) break;
      if (st0 && !((live[0] >> k) & 1)) C[(size_t)row * n_valid + col] = ninf;
      if (st1 && !((live[1] >> k) & 1)) C[(size_t)(row + 8) * n_valid + col] = ninf;
    }
  }
}

// The value column d of a head tile with a value head, which pass 1 of the sampling and Gaussian epilogues parked
// with the policy's columns: bf16 pair 2·(d >> 3) + h of the lane whose columns include d (col0 = 2·(lane % 4) in the
// head's one tile), element d & 1.  That lane widens it to fp32 into values[row + 8h] of the stored rows.  It reads
// the ring rather than acc[]: a run-time index into the accumulators would put them in local memory.
template <typename Slot>
__device__ __forceinline__ void store_values(Slot slot, int d, int row, bool st0, bool st1, float* values) {
  if (values == nullptr || (int)(threadIdx.x & 3) != ((d >> 1) & 3)) return;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const __nv_bfloat162 y = *slot(2 * (d >> 3) + h);
    if (h ? st1 : st0) values[row + 8 * h] = d & 1 ? __high2float(y) : __low2float(y);
  }
}

// The column groups of a multi-discrete head (HeadOut::groups), passed by value with the launch: group g is the
// policy's columns [lo_g, lo_{g+1}), bit j of `starts` is set when column j begins a group (bit 0 included), and the
// last group ends at the policy's width.  n == 0 is the one categorical over every column of the existing entries.
struct HeadGroups {
  uint32_t starts[8] = {};
  int n = 0;
  bool greedy = false;   // rank the logits alone: no noise and no log-probabilities (outputs "actions" and "both")
};

// The log-std of a state-dependent Gaussian head, the layer kernel's last parameter (by value: no upload per call):
// with `state` the head's weight interleaves the mean's and the log-std's rows, and the log-std is clamped to
// [lo, hi]; `squash` passes the actions through tanh.  state == false is the state-independent log_std of the other
// entries.  It is a parameter of its own rather than a member of HeadOut: a larger HeadOut re-schedules the kSample
// instantiations, which never read it.  `det` marks a deterministic actor (TD3 / DDPG) instead: the action is the
// mean, tanh-squashed with `squash`, plus σ·z clamped to [−clip, clip] when σ = `noise` != 0 (deterministic_pass).
struct HeadStd {
  float lo = 0.f, hi = 0.f;
  bool state = false;
  bool squash = false;
  bool det = false;
  float noise = 0.f, clip = 0.f;
};

// The per-row inputs and outputs of an ε-greedy kSample head, the layer kernel's last parameter (by value, like
// HeadStd, and for the same reason: a larger HeadOut re-schedules the other instantiations).  epsilon != null marks
// the head: ε [rows] in, q [rows] and q_max [rows] out beside HeadOut::actions (epsilon_pass).
struct HeadEps {
  const float* epsilon = nullptr;
  float* q = nullptr;
  float* q_max = nullptr;

  HeadEps from_row(size_t r0) const {
    return epsilon ? HeadEps{epsilon + r0, q + r0, q_max + r0} : *this;
  }
};

// The given actions and the entropy output of an evaluating head, the layer kernel's last parameter (by value, like
// HeadEps, and for the same reason).  `actions` != null marks a kSample head that scores int64 group-relative actions
// [rows, max(groups.n, 1)] (evaluate_pass); `gauss_actions` != null marks a kGaussian head that scores fp32 actions
// [rows, d_out] (gaussian_epilogue).  Either writes HeadOut::log_probs and entropy [rows] and draws no noise.
struct HeadEval {
  const int64_t* actions = nullptr;
  const float* gauss_actions = nullptr;
  float* entropy = nullptr;

  // The same inputs and outputs from row r0 on, `per_row` actions per row.
  HeadEval from_row(size_t r0, size_t per_row) const {
    HeadEval e = *this;
    if (actions) e.actions += r0 * per_row;
    if (gauss_actions) e.gauss_actions += r0 * per_row;
    if (entropy) e.entropy += r0;
    return e;
  }
};

// The outputs of a critic head, the layer kernel's last parameter (by value, like HeadEps, and for the same reason).
// q != null marks a kGaussian head with no policy columns whose column 0 is Q(s, a): q [rows] receives it widened to
// fp32.  The second head of a twin also reads q_other [rows], the first head's Q, and stores q_min = min(Q2, Q1)
// (critic_epilogue).  y != null marks the last critic head of a TD target instead: it stores no Q but
// y = r + γ·(1 − d)·(t − α·logp) (t its Q, or the twin's minimum; the α term only with logp) from reward, done and
// logp [rows].  In a kSample head y != null marks a DQN target's target network (dqn_pass): y = r + γ·(1 − d)·q with
// q its value at the action sel [rows] (Double DQN's, chosen by the online network) or at its own greedy action
// (sel null), reading reward[r·rd_stride] and done[r·rd_stride] (2: the interleaved pairs of the pushed forms).
struct HeadQ {
  float* q = nullptr;
  const float* q_other = nullptr;
  float* q_min = nullptr;
  const float* reward = nullptr;
  const float* done = nullptr;
  const float* logp = nullptr;
  float* y = nullptr;
  float gamma = 0.f, alpha = 0.f;
  const int64_t* sel = nullptr;
  int rd_stride = 1;

  // The same outputs from row r0 of the call on.  A TD or DQN target's heads (`scratch`) read and write q, q_other,
  // logp and sel in chunk-sized scratch from the chunk's first row, so only its reward, done and y move.
  HeadQ from_row(size_t r0, bool scratch) const {
    HeadQ h = *this;
    if (scratch) {
      if (y) {
        h.reward += r0 * rd_stride;
        h.done += r0 * rd_stride;
        h.y += r0;
      }
    } else if (q) {
      h.q += r0;
      if (q_other) h.q_other += r0;
      if (q_min) h.q_min += r0;
    }
    return h;
  }
};

// The Bellman target of both target heads: y = r + γ·(1 − d)·t, each operation rounded once in the order torch
// evaluates reward + gamma * (1 - done) * t on fp32 tensors with a Python-float γ (no contraction).
__device__ __forceinline__ float bellman_target(float r, float d, float gamma, float t) {
  return __fadd_rn(r, __fmul_rn(__fmul_rn(gamma, __fsub_rn(1.f, d)), t));
}

// The epilogue of a critic head (HeadQ) in the 64-wide kGaussian instantiation: column 0 of rows row and row + 8, held
// by lane 0 of each quad in acc[0] and acc[2], gets the bias and one rounding to bf16 (layer_pair, as every head) and
// is stored widened to fp32 into q.  A twin's second head also stores q_min = Q2 < Q1 ? Q2 : Q1, so a tie (±0
// included) gives Q1, as torch.minimum of 0-d CPU tensors does, and NaN when either is NaN.  The last head of a TD target
// (hq.y) stores y = r + γ·(1 − d)·t in place of q and q_min, t its Q or that minimum less α·logp when it has logp,
// each operation rounded once in the order of the torch expression (no contraction).  The kernel takes it in place
// of gaussian_epilogue, so the Gaussian heads' code is what it was; the store is rolled.
template <int BLOCK_N>
__device__ __forceinline__ void critic_epilogue(const float (&acc)[BLOCK_N / 2], const __nv_bfloat16* bias, int col0,
                                                int row, bool st0, bool st1, const HeadQ& hq) {
  if (col0 != 0) return;
  __nv_bfloat162 y0, y1;
  layer_pair<false>(acc[0], acc[1], acc[2], acc[3], bias, 0, 1, y0, y1);
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    if (!(h ? st1 : st0)) continue;
    const int r = row + 8 * h;
    const float v = __low2float(h ? y1 : y0);
    float t = v;
    if (hq.q_other != nullptr) {
      const float o = hq.q_other[r];
      t = v != v ? v : v < o ? v : o;
    }
    if (hq.y == nullptr) {
      hq.q[r] = v;
      if (hq.q_other != nullptr) hq.q_min[r] = t;
      continue;
    }
    if (hq.logp != nullptr) t = __fsub_rn(t, __fmul_rn(hq.alpha, hq.logp[r]));
    hq.y[r] = bellman_target(hq.reward[r], hq.done[r], hq.gamma, t);
  }
}

// The end of the group that begins at column lo: the next set bit of `starts` past lo, or d.  The words are indexed
// at compile time, so the bitmap stays in the kernel's parameters.
__device__ __forceinline__ int group_end(const uint32_t (&starts)[8], int lo, int d) {
  int hi = d;
#pragma unroll
  for (int w = 7; w >= 0; --w) {
    const int s = lo + 1 - 32 * w;   // bits >= s of word w are the columns past lo
    const uint32_t b = s <= 0 ? starts[w] : s >= 32 ? 0u : starts[w] & (~0u << s);
    if (b) hi = 32 * w + __ffs(b) - 1;
  }
  return hi;
}

// The grouped pass of sample_epilogue (groups.n > 0) over the bf16 pairs that its pass 1 parked in the ring.  Each
// group is the rolled pass of the single categorical over the group's columns alone: a per-thread max of the live
// columns in [lo, hi) and a quad max, then one pass that ranks y + Gumbel noise (y alone when greedy) in
// torch.argmax order and sums exp(y - m), each in the single categorical's per-thread and quad order, so a group is
// bit for bit that head under the mask legal ∧ (column in the group).  The loop over groups is uniform across the warp,
// so every shuffle is converged.  A pair that straddles a group boundary draws its Philox words once: x[] keeps the
// last pair's.  actions[row·n + g] is the group-relative action (0 when the group's ranked values are all -inf), and
// log_probs[row] the fp32 sum of the groups' log-probabilities in group order, starting from group 0's.  With C, the
// bf16 logits of "both" are stored from the ring, -inf in illegal columns, as greedy_epilogue stores them.
template <int BLOCK_N, typename Slot>
__device__ __forceinline__ void group_pass(Slot slot, const ColBits<BLOCK_N> (&live)[2], const HeadGroups& groups,
                                           int d, int col0, int row, bool st0, bool st1, __nv_bfloat16* C,
                                           int64_t* actions, float* log_probs, uint64_t seed, uint64_t row_base) {
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const bool draw = !groups.greedy;
  const int G = groups.n;
  float lp[2] = {0.f, 0.f};
  uint2 x[2] = {make_uint2(0u, 0u), make_uint2(0u, 0u)};
  int drawn = -1;   // the pair whose Philox words x[] hold
  int lo = 0;
#pragma unroll 1
  for (int g = 0; g < G; ++g) {
    const int hi = group_end(groups.starts, lo, d);
    const int j0 = max(0, (lo - col0 + 6) >> 3);   // the first pair of the thread with col0 + 8j + 1 >= lo
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll 1
    for (int j = j0; j < BLOCK_N / 8; ++j) {
      const int col = col0 + 8 * j;
      if (col >= hi) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float v = c ? __high2float(y) : __low2float(y);
          if (col + c >= lo && col + c < hi && ((live[h] >> (2 * j + c)) & 1) && v > mx[h]) mx[h] = v;
        }
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
    float best[2] = {-INFINITY, -INFINITY}, best_y[2] = {NAN, NAN}, sum[2] = {0.f, 0.f};
    int best_col[2] = {INT_MAX, INT_MAX};
#pragma unroll 1
    for (int j = j0; j < BLOCK_N / 8; ++j) {
      const int col = col0 + 8 * j;
      if (col >= hi) break;
      if (draw && j != drawn) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t i = row_base + (uint64_t)(row + 8 * h);
          const uint4 w = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)col >> 1, 0u), key);
          x[h] = make_uint2(w.x, w.y);
        }
        drawn = j;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (col + c < lo || col + c >= hi || !((live[h] >> (2 * j + c)) & 1)) continue;
          const float v = c ? __high2float(y) : __low2float(y);
          const float s = draw ? v + gumbel_of(c ? x[h].y : x[h].x) : v;
          if (argmax_before(s, col + c, best[h], best_col[h])) {
            best[h] = s;
            best_col[h] = col + c;
            best_y[h] = v;
          }
          if (draw) sum[h] += v == mx[h] ? 1.f : expf(v - mx[h]);
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
      const float t = best_y[h] - mx[h] - logf(sum[h]);
      lp[h] = g == 0 ? t : lp[h] + t;
    }
    if ((threadIdx.x & 3) == 0 && actions != nullptr) {
      if (st0) actions[(size_t)row * G + g] = best[0] == -INFINITY ? 0 : best_col[0] - lo;
      if (st1) actions[(size_t)(row + 8) * G + g] = best[1] == -INFINITY ? 0 : best_col[1] - lo;
    }
    lo = hi;
  }
  if (draw && (threadIdx.x & 3) == 0) {
    if (st0) log_probs[row] = lp[0];
    if (st1) log_probs[row + 8] = lp[1];
  }
  if (C == nullptr) return;
  const __nv_bfloat16 ninf = __ushort_as_bfloat16((unsigned short)0xFF80u);
  const bool pairs = (d & 1) == 0 && ((uintptr_t)C & 3) == 0;
#pragma unroll 1
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= d) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!(h ? st1 : st0)) continue;
      __nv_bfloat162 y = *slot(2 * j + h);
      if (!((live[h] >> (2 * j)) & 1)) y.x = ninf;
      if (!((live[h] >> (2 * j + 1)) & 1)) y.y = ninf;
      __nv_bfloat16* p = C + (size_t)(row + 8 * h) * d + col;
      if (pairs) {
        *reinterpret_cast<__nv_bfloat162*>(p) = y;
      } else {
        p[0] = y.x;
        if (col + 1 < d) p[1] = y.y;
      }
    }
  }
}

// The evaluating pass of sample_epilogue (HeadEval::actions != null) over the bf16 pairs that its pass 1 parked in the
// ring: the log-probability and the entropy of given actions.  The single categorical is one group over the policy's
// d columns (groups.n == 0: group_end gives d).  Each group is group_pass's with the action read instead of drawn: a
// per-thread max of the live columns in [lo, hi) and a quad max m, then S = Σ (y == m ? 1 : expf(y − m)) and
// T = Σ w·(y − m) (w the term of S, one fused multiply-add; a -inf column adds to neither) in group_pass's per-thread
// and quad order, so S, m and the log-probability of the sampled action are group_pass's (and the single rolled pass's)
// bits.  Every lane of a quad reads taken[r, g] of its two rows; the lane whose columns include lo + a reads y_a from
// its slot (-inf when illegal) and shfl.xor shares it across the quad.  lp_g is NaN for a ∉ [0, hi − lo) or m == -inf
// (no legal column, or only -inf ones), -inf for an illegal column, else y_a − m − logf(S); H_g is NaN in the first two
// cases, else logf(S) − T / S.  log_probs[r] and entropy[r] are the fp32 sums over groups in group order, starting from
// group 0's term.
template <int BLOCK_N, typename Slot>
__device__ __forceinline__ void evaluate_pass(Slot slot, const ColBits<BLOCK_N> (&live)[2], const HeadGroups& groups,
                                              int d, int col0, int row, bool st0, bool st1, const int64_t* taken,
                                              float* log_probs, float* entropy) {
  const int G = groups.n > 0 ? groups.n : 1;
  const int lane = threadIdx.x & 31;
  float lp[2] = {0.f, 0.f}, ent[2] = {0.f, 0.f};
  int lo = 0;
#pragma unroll 1
  for (int g = 0; g < G; ++g) {
    const int hi = group_end(groups.starts, lo, d);
    const int j0 = max(0, (lo - col0 + 6) >> 3);   // the first pair of the thread with col0 + 8j + 1 >= lo
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll 1
    for (int j = j0; j < BLOCK_N / 8; ++j) {
      const int col = col0 + 8 * j;
      if (col >= hi) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float v = c ? __high2float(y) : __low2float(y);
          if (col + c >= lo && col + c < hi && ((live[h] >> (2 * j + c)) & 1) && v > mx[h]) mx[h] = v;
        }
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
    float sum[2] = {0.f, 0.f}, t[2] = {0.f, 0.f};
#pragma unroll 1
    for (int j = j0; j < BLOCK_N / 8; ++j) {
      const int col = col0 + 8 * j;
      if (col >= hi) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (col + c < lo || col + c >= hi || !((live[h] >> (2 * j + c)) & 1)) continue;
          const float v = c ? __high2float(y) : __low2float(y);
          const float w = v == mx[h] ? 1.f : expf(v - mx[h]);
          sum[h] += w;
          if (v != -INFINITY) t[h] = __fmaf_rn(w, v - mx[h], t[h]);
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // the action's column (-1: out of range); every lane of the quad reads the same row's
      const int64_t a = (h ? st1 : st0) ? taken[(size_t)(row + 8 * h) * G + g] : -1;
      const int col = a >= 0 && a < hi - lo ? lo + (int)a : -1;
      const int owner = col < 0 ? lane & 3 : (col >> 1) & 3;
      float ya = -INFINITY;
      if (col >= 0 && owner == (lane & 3)) {
        const int j = (col - col0) >> 3, c = col & 1;
        const __nv_bfloat162 y = *slot(2 * j + h);
        if ((live[h] >> (2 * j + c)) & 1) ya = c ? __high2float(y) : __low2float(y);
      }
#pragma unroll
      for (int m = 1; m <= 2; m <<= 1) {
        sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], m);
        t[h] += __shfl_xor_sync(0xffffffffu, t[h], m);
        const float oy = __shfl_xor_sync(0xffffffffu, ya, m);
        if ((lane ^ owner) & m) ya = oy;   // the partner is nearer the owner: after m = 1, 2 every lane holds y_a
      }
      const bool bad = col < 0 || mx[h] == -INFINITY;
      const float l = logf(sum[h]);
      const float lpg = bad ? NAN : ya == -INFINITY ? -INFINITY : ya - mx[h] - l;
      const float hg = bad ? NAN : l - t[h] / sum[h];
      lp[h] = g == 0 ? lpg : lp[h] + lpg;
      ent[h] = g == 0 ? hg : ent[h] + hg;
    }
    lo = hi;
  }
  if ((threadIdx.x & 3) == 0) {
    if (st0) {
      log_probs[row] = lp[0];
      entropy[row] = ent[0];
    }
    if (st1) {
      log_probs[row + 8] = lp[1];
      entropy[row + 8] = ent[1];
    }
  }
}

// The ε-greedy pass of sample_epilogue (epsilon != null) over the bf16 pairs that its pass 1 parked in the ring: a
// Q-network's actor.  For each of the thread's rows r = row + 8h (global row i = row_base + r):
//   * the greedy action g: torch.argmax of the live columns (argmax_before; 0 when their values are all -inf or there
//     are none), ranked in the greedy epilogue's per-thread and quad order;
//   * the coin: u = (2·(x >> 9) + 1)·2^-24 of word 0 of Philox counter (i, 0, 3), drawn once per row by lane h of the
//     quad's pair (lanes 0, 2 draw row's, lanes 1, 3 row + 8's) and shared by shfl.xor; the row explores iff
//     u < epsilon[r] in fp32 (so ε <= 0 and a NaN ε never explore);
//   * an exploring row, and only such a row, draws Philox word c of counter (i, col >> 1, 2) for each pair (col,
//     col + 1), and takes the live column with the largest word, ties to the lower column (0 when none is live).  The
//     rank key is (word << 32) | ~col, so 0 means "no live column" and a larger key wins.
// Lane 0 of the quad stores actions[r], q[r] = the masked Q-value of the action taken and q_max[r] = that of g, both
// widened exactly from bf16 (an illegal column's is -inf).
template <int BLOCK_N, typename Slot>
__device__ __forceinline__ void epsilon_pass(Slot slot, const ColBits<BLOCK_N> (&live)[2], int d, int col0, int row,
                                             bool st0, bool st1, const float* epsilon, int64_t* actions, float* q,
                                             float* q_max, uint64_t seed, uint64_t row_base) {
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  float best[2] = {-INFINITY, -INFINITY};
  int best_col[2] = {INT_MAX, INT_MAX};
#pragma unroll 1
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= d) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float v = c ? __high2float(y) : __low2float(y);
        if (((live[h] >> (2 * j + c)) & 1) && argmax_before(v, col + c, best[h], best_col[h])) {
          best[h] = v;
          best_col[h] = col + c;
        }
      }
    }
  }
  const int hc = threadIdx.x & 1;   // the row whose coin this lane draws
  int mine = 0;
  if (hc ? st1 : st0) {
    const uint64_t i = row_base + (uint64_t)(row + 8 * hc);
    const uint32_t x = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), 0u, 3u), key).x;
    mine = (float)(2u * (x >> 9) + 1u) * 5.9604644775390625e-8f < epsilon[row + 8 * hc];
  }
  const int other = __shfl_xor_sync(0xffffffffu, mine, 1);
  const bool explore[2] = {(hc ? other : mine) != 0, (hc ? mine : other) != 0};
  unsigned long long rank[2] = {0ull, 0ull};
  float ey[2] = {-INFINITY, -INFINITY};
  if (explore[0] || explore[1]) {
#pragma unroll 1
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int col = col0 + 8 * j;
      if (col >= d) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!explore[h]) continue;
        const uint64_t i = row_base + (uint64_t)(row + 8 * h);
        const uint4 x = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)col >> 1, 2u), key);
        const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const unsigned long long k = (unsigned long long)(c ? x.y : x.x) << 32 | (uint32_t)~(col + c);
          if (((live[h] >> (2 * j + c)) & 1) && k > rank[h]) {
            rank[h] = k;
            ey[h] = c ? __high2float(y) : __low2float(y);
          }
        }
      }
    }
  }
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
      const unsigned long long ok = __shfl_xor_sync(0xffffffffu, rank[h], m);
      const float oy = __shfl_xor_sync(0xffffffffu, ey[h], m);
      if (ok > rank[h]) {
        rank[h] = ok;
        ey[h] = oy;
      }
    }
  }
  if ((threadIdx.x & 3) == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!(h ? st1 : st0)) continue;
      const int g = best[h] == -INFINITY ? 0 : best_col[h];
      const int e = rank[h] == 0 ? 0 : (int)~(uint32_t)rank[h];
      actions[row + 8 * h] = explore[h] ? e : g;
      q[row + 8 * h] = explore[h] ? ey[h] : best[h];
      q_max[row + 8 * h] = best[h];
    }
  }
}

// The DQN target's pass of sample_epilogue (hq.y != null) over the bf16 pairs that its pass 1 parked in the ring: the
// target network's head.  For each of the thread's rows r = row + 8h:
//   * the action a: hq.sel[r] (Double DQN: the online network's greedy action, which every lane of the quad reads), or
//     with sel null (DQN) the greedy action of this head's live columns, ranked as epsilon_pass ranks g (argmax_before
//     in the greedy epilogue's per-thread and quad order; 0 when their values are all -inf or there are none);
//   * q: the lane whose columns include a reads its parked value with no live-bit test, so q is the UNMASKED target
//     value widened exactly (a terminal state with no legal action reads column 0, and done = 1 then gives y = r
//     rather than 0·(−inf)), and shfl.xor shares it across the quad, as evaluate_pass shares y_a;
//   * lane 0 of the quad stores y[r] = bellman_target(reward[r·s], done[r·s], γ, q), s = hq.rd_stride.
template <int BLOCK_N, typename Slot>
__device__ __forceinline__ void dqn_pass(Slot slot, const ColBits<BLOCK_N> (&live)[2], int d, int col0, int row,
                                         bool st0, bool st1, const HeadQ& hq) {
  const int lane = threadIdx.x & 31;
  int a[2] = {0, 0};
  if (hq.sel != nullptr) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (h ? st1 : st0) a[h] = (int)hq.sel[row + 8 * h];
  } else {
    float best[2] = {-INFINITY, -INFINITY};
    int best_col[2] = {INT_MAX, INT_MAX};
#pragma unroll 1
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int col = col0 + 8 * j;
      if (col >= d) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float v = c ? __high2float(y) : __low2float(y);
          if (((live[h] >> (2 * j + c)) & 1) && argmax_before(v, col + c, best[h], best_col[h])) {
            best[h] = v;
            best_col[h] = col + c;
          }
        }
      }
    }
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
      a[h] = best[h] == -INFINITY ? 0 : best_col[h];
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int owner = (a[h] >> 1) & 3;
    float q = 0.f;
    if (owner == (lane & 3)) {
      const __nv_bfloat162 y = *slot(2 * ((a[h] - col0) >> 3) + h);
      q = a[h] & 1 ? __high2float(y) : __low2float(y);
    }
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      const float oq = __shfl_xor_sync(0xffffffffu, q, m);
      if ((lane ^ owner) & m) q = oq;   // the partner is nearer the owner: after m = 1, 2 every lane holds q
    }
    if ((lane & 3) == 0 && (h ? st1 : st0)) {
      const size_t r = (size_t)(row + 8 * h) * hq.rd_stride;
      hq.y[row + 8 * h] = bellman_target(hq.reward[r], hq.done[r], hq.gamma, q);
    }
  }
}

// The sampling epilogue of a head tile (HeadKind::kSample): rows r = row and row + 8 of the thread, global rows
// row_base + r.  Pass 1 (unrolled over the accumulators) rounds the logits once, parks them as bf16 pairs in the TMA
// ring as gaussian_epilogue does, and takes each row's largest logit m across the quad (NaN skipped: it reaches the sum
// instead); pass 2 is a rolled loop, so the Philox code is not repeated BLOCK_N / 8 times (the 256-wide head had
// 17 576 instructions with it unrolled, and any code added to it, even code the unmasked call skips, made that call
// 3 % slower, H100 80GB HBM3, 700 W).  It draws one
// Philox call per column pair < n_valid and row, ranks fp32(logit + noise) in torch.argmax order and sums
// exp(logit - m) without a running rescale.  A logit equal to m adds 1 without an exp, so an all -inf (or a +inf)
// maximum never forms exp(inf - inf): such rows end with a NaN log-probability, as in torch, and -inf logits beside a
// finite m add 0.  With a legal-action mask both passes skip illegal columns (live_columns): a -inf logit adds 0 beside
// a finite or +inf m and never wins the Gumbel-max while a legal logit is finite, so this is the sample of
// logits.masked_fill(~legal, -inf).  A row whose ranked values are all -inf (every legal logit -inf, or no legal
// column) takes action 0 with a NaN log-probability, as torch does.
// With a value head (values != null) the tile holds n_valid = d + 1 columns: the policy's d, then the value column d.
// Pass 1 parks column d with the rest; everything ranked, drawn, summed or masked stops at d; store_values reads it.
// A multi-discrete head (groups.n > 0) takes group_pass in place of the rolled pass: the greedy one as well, whose
// logits (C, unless null) it also stores.  An ε-greedy head (epsilon != null) takes epsilon_pass in its place, and an
// evaluating head (ev.actions != null), grouped or not, evaluate_pass, and a DQN target's target network (hq.y != null)
// dqn_pass.  The single categorical's rolled pass stays as it is.
template <int BLOCK_N, int STAGES>
__device__ __forceinline__ void sample_epilogue(const float (&acc)[BLOCK_N / 2], const __nv_bfloat16* bias, int col0,
                                                int n_valid, int row, bool st0, bool st1, int64_t* actions,
                                                float* log_probs, const uint8_t* mask, uint64_t seed,
                                                uint64_t row_base, float* values, const HeadGroups& groups,
                                                __nv_bfloat16* C, const float* epsilon, float* q, float* q_max,
                                                const HeadEval& ev, const HeadQ& hq) {
  using S = MlpSmem<BLOCK_N, STAGES>;
  static_assert(BLOCK_N / 64 <= STAGES, "each warp's bf16 pairs fill its 16 A rows of BLOCK_N / 64 stages");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // pair w (= 2j + h) of a lane parked as in gaussian_epilogue: stage w / 16, the warp's own 16 A rows, word
  // (w % 16)·32 + lane
  uint8_t* mine = smem + (threadIdx.x >> 5) * 16 * 128 + (threadIdx.x & 31) * 4;
  auto slot = [&](int w) { return reinterpret_cast<__nv_bfloat162*>(mine + (w >> 4) * S::kStageBytes + (w & 15) * 128); };
  const int d = n_valid - (values != nullptr);   // the policy's columns
  ColBits<BLOCK_N> live[2];
  live_columns<BLOCK_N>(mask, row, col0, d, st0, st1, live);
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= n_valid) continue;
    __nv_bfloat162 y[2];   // y[h]: columns (col, col + 1) of row + 8h
    layer_pair<false>(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col, n_valid, y[0], y[1]);
    *slot(2 * j) = y[0];
    *slot(2 * j + 1) = y[1];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float v = q & 1 ? __high2float(y[q >> 1]) : __low2float(y[q >> 1]);
      if (((live[q >> 1] >> (2 * j + (q & 1))) & 1) && v > mx[q >> 1]) mx[q >> 1] = v;
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
  if (ev.actions != nullptr) {
    evaluate_pass<BLOCK_N>(slot, live, groups, d, col0, row, st0, st1, ev.actions, log_probs, ev.entropy);
    store_values(slot, d, row, st0, st1, values);
    return;
  }
  if (groups.n > 0) {
    group_pass<BLOCK_N>(slot, live, groups, d, col0, row, st0, st1, C, actions, log_probs, seed, row_base);
    store_values(slot, d, row, st0, st1, values);
    return;
  }
  if (epsilon != nullptr) {
    epsilon_pass<BLOCK_N>(slot, live, d, col0, row, st0, st1, epsilon, actions, q, q_max, seed, row_base);
    return;
  }
  if (hq.y != nullptr) {
    dqn_pass<BLOCK_N>(slot, live, d, col0, row, st0, st1, hq);
    return;
  }
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  float best[2] = {-INFINITY, -INFINITY}, best_y[2] = {NAN, NAN}, sum[2] = {0.f, 0.f};
  int best_col[2] = {INT_MAX, INT_MAX};
#pragma unroll 1
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= d) break;   // a pair wholly past the policy draws no noise
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint64_t i = row_base + (uint64_t)(row + 8 * h);
      const uint4 x = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)col >> 1, 0u), key);
      // (column d of a value head is never live: live_columns stops at d)
      const __nv_bfloat162 y = *slot(2 * j + h);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (!((live[h] >> (2 * j + c)) & 1)) continue;
        const float v = c ? __high2float(y) : __low2float(y);
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
  store_values(slot, d, row, st0, st1, values);
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
      actions[row] = best[0] == -INFINITY ? 0 : best_col[0];
      log_probs[row] = best_y[0] - mx[0] - logf(sum[0]);
    }
    if (st1) {
      actions[row + 8] = best[1] == -INFINITY ? 0 : best_col[1];
      log_probs[row + 8] = best_y[1] - mx[1] - logf(sum[1]);
    }
  }
}

// The deterministic actor's pass of gaussian_epilogue (HeadStd::det) over the bf16 pairs its pass 1 parked: one rolled
// step per column pair < d.  t = tanhf(μ) with sd.squash, μ otherwise; when sd.noise != 0 one Philox call per pair and
// row draws the Gaussian head's z (word col & 1 of counter (i, col >> 1, 1)), n = σ·z rounded once and clamped to
// [−clip, clip], and t = t + n rounded once (no FMA contraction: the same rounding as the torch body); with sd.squash t
// is then clamped to [−1, 1].  The clamps are compares, not fminf / fmaxf, so a NaN μ stays NaN.  σ = 0 draws no
// Philox word.  Stored as in the sampling branch: float2 where the row stride and the base allow, scalars otherwise.
template <int BLOCK_N, typename Slot>
__device__ __forceinline__ void deterministic_pass(Slot slot, int col0, int d, int row, bool st0, bool st1,
                                                   float* actions, uint2 key, uint64_t row_base, const HeadStd& sd,
                                                   bool pairs) {
  const float s = sd.noise, c = sd.clip;
#pragma unroll 1
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= d) break;
    const bool has1 = col + 1 < d;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __nv_bfloat162 y = *slot(2 * j + h);
      float a[2] = {__low2float(y), __high2float(y)};
      if (sd.squash) {
        a[0] = tanhf(a[0]);
        a[1] = tanhf(a[1]);
      }
      if (s != 0.f) {
        const uint64_t i = row_base + (uint64_t)(row + 8 * h);
        const uint4 x = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)col >> 1, 1u), key);
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const float z = normcdfinvf((float)(2u * ((k ? x.y : x.x) >> 9) + 1u) * 5.9604644775390625e-8f);
          float n = __fmul_rn(s, z);
          n = n < -c ? -c : n > c ? c : n;
          a[k] = __fadd_rn(a[k], n);
        }
      }
      if (sd.squash) {
#pragma unroll
        for (int k = 0; k < 2; ++k) a[k] = a[k] < -1.f ? -1.f : a[k] > 1.f ? 1.f : a[k];
      }
      if (!(h ? st1 : st0)) continue;
      float* p = actions + (size_t)(row + 8 * h) * d + col;
      if (pairs) {
        *reinterpret_cast<float2*>(p) = make_float2(a[0], a[1]);
      } else {
        p[0] = a[0];
        if (has1) p[1] = a[1];
      }
    }
  }
}

// The Gaussian epilogue of a head tile (HeadKind::kGaussian): rows r = row and row + 8 of the thread, global rows
// row_base + r.  Only its first part is unrolled over the accumulators, so that the Philox and Φ⁻¹ code is not repeated
// BLOCK_N / 8 times: it rounds the logits once (layer_pair: μ, the value ktb_mlp_bf16_policy stores) and parks them as
// bf16 pairs in the TMA ring, each warp in the 16 A rows of every stage that only its own accumulator rows are made of:
// once the warp's wgmmas are waited for nothing reads or writes them again (every load has landed, and no other warp's
// wgmma reads those rows).  A rolled loop then makes one pass over the column pairs < n_valid: one Philox call per pair
// and row (counter word 3 = 1: never the Gumbel stream's uniforms), z = Φ⁻¹(u) (normcdfinvf, no fast-math; u is never
// 0.5, so z != 0), the action μ + σ·z rounded twice (no FMA contraction), stored as float2 where the row stride and the
// base allow and as scalars otherwise, and Σ (0.5·z² + log_std) per row for the log-probability, which does not read μ.
// With a value head (values != null) the tile holds n_valid = d + 1 columns, as in sample_epilogue: the rolled pass,
// the actions' row stride and the log-density's constant cover the policy's d columns only.
// An evaluating head (ev.gauss_actions != null) takes a third rolled pass in place of the sampling one: it draws no
// noise, reads the given actions a [rows, d] (float2 where the row stride and the base allow, as the action stores),
// sums 0.5·z² + log_std with z = __fdiv_rn(__fsub_rn(a, μ), expf(log_std)) in the sampling pass's per-thread and quad
// order, and stores ev.entropy[row] = Σ (log_std + 0.5) + d·0.5·log(2π), summed in the same order for every row.
// A state-dependent head (sd.state) takes a rolled pass of its own after the same pass 1: its d = 2·d_out policy
// columns interleave the mean and the log-std, so pair (2a, 2a + 1) of a thread is (μ_a, ℓ_a) of action a, one parked
// bf16x2 slot.  ℓ is clamped to [sd.lo, sd.hi] by compares (a NaN stays NaN), σ = expf(ℓc), z is Philox word a & 1
// of counter (i, a >> 1, 1) (the noise of action a in the head above), u = μ + σ·z rounded as above, and the action is
// tanhf(u) with sd.squash, u without; the row sums 0.5·z² + ℓc, plus 2·(log 2 − |u| − log1p(e^−2|u|)) =
// −log(1 − tanh²u) with sd.squash, over its d_out actions.
// A deterministic actor (sd.det) takes deterministic_pass after the same pass 1 and returns: it stores no
// log-probabilities.
template <int BLOCK_N, int STAGES>
__device__ __forceinline__ void gaussian_epilogue(const float (&acc)[BLOCK_N / 2], const __nv_bfloat16* bias, int col0,
                                                  int n_valid, int row, bool st0, bool st1, const float* log_std,
                                                  float* actions, float* log_probs, uint64_t seed, uint64_t row_base,
                                                  float* values, const HeadStd& sd, const HeadEval& ev) {
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
    layer_pair<false>(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], bias, col, n_valid, *slot(2 * j),
                      *slot(2 * j + 1));
  }
  const int d = n_valid - (values != nullptr);   // the policy's columns
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const bool pairs = (d & 1) == 0 && ((uintptr_t)actions & 7) == 0;
  if (sd.det) {   // no log-probabilities and no value head
    deterministic_pass<BLOCK_N>(slot, col0, d, row, st0, st1, actions, key, row_base, sd, pairs);
    return;
  }
  const int d_act = sd.state ? d >> 1 : d;   // the actions per row
  float sum[2] = {0.f, 0.f};
#pragma unroll 1
  for (int j = 0; sd.state && j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= d) break;   // d is even: col + 1 < d
    const int a = col >> 1;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __nv_bfloat162 y = *slot(2 * j + h);
      const float l = __high2float(y);
      const float lc = l < sd.lo ? sd.lo : l > sd.hi ? sd.hi : l;   // not fminf / fmaxf: they drop a NaN
      const uint64_t i = row_base + (uint64_t)(row + 8 * h);
      const uint4 x = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)a >> 1, 1u), key);
      const float z = normcdfinvf((float)(2u * ((a & 1 ? x.y : x.x) >> 9) + 1u) * 5.9604644775390625e-8f);
      const float u = __fadd_rn(__low2float(y), __fmul_rn(expf(lc), z));
      float t = 0.5f * z * z + lc;
      if (sd.squash) {
        const float au = fabsf(u);
        t += 2.f * (0.693147180559945309f - au - log1pf(expf(-2.f * au)));
      }
      sum[h] += t;
      if (h ? st1 : st0) actions[(size_t)(row + 8 * h) * d_act + a] = sd.squash ? tanhf(u) : u;
    }
  }
#pragma unroll 1
  for (int j = 0; !sd.state && ev.gauss_actions == nullptr && j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= d) break;   // a pair wholly past the policy draws no noise
    const __nv_bfloat162 y[2] = {*slot(2 * j), *slot(2 * j + 1)};
    const bool has1 = col + 1 < d;
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
      float* p = actions + (size_t)(row + 8 * h) * d + col;
      if (pairs) {
        *reinterpret_cast<float2*>(p) = make_float2(a[0], a[1]);
      } else {
        p[0] = a[0];
        if (has1) p[1] = a[1];
      }
    }
  }
  const float* taken = ev.gauss_actions;
  const bool taken_pairs = (d & 1) == 0 && ((uintptr_t)taken & 7) == 0;
  float ent = 0.f;
#pragma unroll 1
  for (int j = 0; taken != nullptr && j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= d) break;
    const __nv_bfloat162 y[2] = {*slot(2 * j), *slot(2 * j + 1)};
    const bool has1 = col + 1 < d;
    const float ls[2] = {log_std[col], has1 ? log_std[col + 1] : 0.f};
    const float sg[2] = {expf(ls[0]), expf(ls[1])};
    ent += ls[0] + 0.5f;
    if (has1) ent += ls[1] + 0.5f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!(h ? st1 : st0)) continue;
      const float* p = taken + (size_t)(row + 8 * h) * d + col;
      float a[2];
      if (taken_pairs) {
        const float2 t = *reinterpret_cast<const float2*>(p);
        a[0] = t.x;
        a[1] = t.y;
      } else {
        a[0] = p[0];
        a[1] = has1 ? p[1] : 0.f;
      }
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float z = __fdiv_rn(__fsub_rn(a[c], c ? __high2float(y[h]) : __low2float(y[h])), sg[c]);
        if (c == 0 || has1) sum[h] += 0.5f * z * z + ls[c];
      }
    }
  }
  store_values(slot, d, row, st0, st1, values);
  // the 4 lanes of a quad hold the columns of the same two rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], m);
  }
  if (taken != nullptr) {
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) ent += __shfl_xor_sync(0xffffffffu, ent, m);
  }
  if ((threadIdx.x & 3) == 0) {
    const float c = (float)d_act * 0.918938533204672742f;   // d_out·0.5·log(2π)
    if (st0) log_probs[row] = -sum[0] - c;
    if (st1) log_probs[row + 8] = -sum[1] - c;
    if (taken != nullptr && st0) ev.entropy[row] = ent + c;
    if (taken != nullptr && st1) ev.entropy[row + 8] = ent + c;
  }
}

// What a layer's epilogue computes: the hidden layers' activation, or the head each entry point names.
enum class HeadKind {
  kHidden,     // bf16 relu(A · Bᵀ + bias) of full tiles (layers 1 and 2)
  kGreedy,     // bf16 logits and/or int64 argmax actions (unrolled; the single categorical)
  kSample,     // the rolled categorical head: Gumbel-max int64 actions and fp32 log_probs, or with groups (HeadGroups)
               // greedy or Gumbel-max actions per group, with the logits of "both" or the summed log_probs, or with
               // epsilon ε-greedy actions and their fp32 Q-values, or with hq.y a DQN target
  kGaussian,   // fp32 actions [rows, d_out] (gauss_actions) drawn with log_std, and fp32 log_probs
};

// The outputs of a layer launch.  A hidden layer stores only its bf16 activation, in `logits`.  Pointers the head
// kind does not store are null.  Row r of the launch draws the noise of global row row_base + r.  `mask`, unless null,
// is the greedy or sampling head's legal-action mask [rows, d_out] (nonzero byte: legal), a runtime input of the same
// instantiations.  `values`, unless null, marks a sampling or Gaussian head with a value head: the head's weight has
// d_out + 1 rows (the policy's, then the critic's), and column d_out of each stored row goes to values[row] in fp32.
// `groups`, with groups.n > 0, marks a multi-discrete kSample head: actions is [rows, groups.n].
struct HeadOut {
  void* logits = nullptr;
  int64_t* actions = nullptr;
  float* log_probs = nullptr;
  uint64_t seed = 0, row_base = 0;
  const float* log_std = nullptr;
  float* gauss_actions = nullptr;
  const uint8_t* mask = nullptr;
  float* values = nullptr;
  HeadGroups groups;

  // The same outputs from row r0 of the call on (d_out: the policy's width).
  HeadOut from_row(size_t r0, int d_out) const {
    HeadOut h = *this;
    if (logits) h.logits = static_cast<__nv_bfloat16*>(logits) + r0 * d_out;
    if (actions) h.actions += r0 * (groups.n > 0 ? groups.n : 1);
    if (log_probs) h.log_probs += r0;
    if (gauss_actions) h.gauss_actions += r0 * d_out;
    if (mask) h.mask += r0 * d_out;
    if (values) h.values += r0;
    h.row_base += r0;
    return h;
  }
};

// One MLP layer: C[:, col] = act(A · Bᵀ + bias[col]) for col < n_valid (C = out.logits, n_valid columns), with the
// bias (unless null) added to the fp32 accumulator and the sum rounded once to bf16 (nn.Linear / F.linear).  One
// output tile per CTA; blockIdx.x walks N, so the CTAs of one 128-row block run side by side and read their A tile from
// L2 once.  Only rows < rows (A's row count) are stored.  KIND picks the epilogue at compile time:
//   kHidden (BLOCK_N = 256): C = relu(...), every tile full (store_tile);
//   kGreedy: logits and/or actions[row] = the argmax of the row's ROUNDED logits (greedy_epilogue);
//   kGreedy and kSample with out.mask: what the head computes from logits.masked_fill(~legal, -inf);
//   kSample: the action of global row i = row_base + row is the argmax of fp32(logit_j + g_j) with g_j the Gumbel
//     noise of Philox word j & 1 of counter (i, j >> 1) under `seed` (include/ktb200.h), and log_probs[row] =
//     log_softmax(logits)[action] in fp32 (sample_epilogue);
//   kGaussian: gauss_actions[row, j] = logit_j + exp(log_std_j)·z_j with z_j = Φ⁻¹(u) of Philox word j & 1 of counter
//     (i, j >> 1, 1), and log_probs[row] the diagonal Normal's log-density of that action (gaussian_epilogue);
//   kGaussian with sd.state: μ and the clamped log-std from the interleaved columns (2a, 2a + 1), optionally
//     tanh-squashed actions, and the log-density with its tanh correction (gaussian_epilogue); n_valid = 2·d_out, and
//     a value head's column is 2·d_out;
//   kSample and kGaussian with out.values: n_valid = d_out + 1, and values[row] = fp32(column d_out) (store_values);
//   kSample with out.groups: one greedy or sampled action per group of columns into actions[row, g], the summed
//     log-probability of the sampled ones, and the logits of a greedy head that stores them (group_pass);
//   kSample with eg.epsilon: the ε-greedy action of each row with the Q-values of the taken and the greedy action
//     (epsilon_pass);
//   kSample with hq.y: a DQN target's target network, y[row] = r + γ·(1 − d)·q with q its unmasked value at the
//     online network's action hq.sel[row] or at its own (masked) greedy action (dqn_pass);
//   kSample with ev.actions and kGaussian with ev.gauss_actions: the log-probability and the entropy of given actions
//     (evaluate_pass, gaussian_epilogue);
//   kGaussian with sd.det: gauss_actions[row, j] = the deterministic actor's action, tanh(logit_j) (or logit_j) plus
//     clipped noise, and no log_probs (deterministic_pass);
//   kGaussian with hq.q: a critic, n_valid = 1: hq.q[row] = fp32(logit_0), and a twin's second head also hq.q_min[row]
//     (critic_epilogue); with hq.y the last critic of a TD target, which stores the target y[row] instead.
// A critic's layer 1 (kHidden) takes its A operand from two maps: K blocks < kb_split from maps_a.m[0] (the
// observation rows), the last from maps_a.m[1] (the action tile); every other launch has kb_split = K / 64 and never
// reads m[1].
// A head runs in the smallest of 64 / 128 / 256 that holds d_out = n_valid, so that one CTA owns whole rows
// (gridDim.x == 1) and the argmax never leaves it.  Columns >= n_valid hold TMA zero fill: they are never stored and
// never an action.
// `bias` is deliberately not __restrict__: with it the compiler reads the bias through the non-coherent cache in
// batches ahead of the stores, and a biased hidden layer takes 3 % longer (H100 80GB HBM3, 700 W).
// The A operand's maps of a layer launch, one kernel parameter: m[1] is read only by a critic's layer 1.  One object
// rather than two parameters: with the second map a parameter of its own, taking its address made ptxas keep the
// Gaussian epilogue's shared-memory addresses out of registers (the 256-wide instantiation grew by a quarter).
struct AMaps {
  CUtensorMap m[2];
};

template <int BLOCK_N, int STAGES, HeadKind KIND>
__global__ void __launch_bounds__(kMlpThreads, 1)
    mlp_layer_wgmma_kernel(const __grid_constant__ AMaps maps_a, const __grid_constant__ CUtensorMap map_b,
                           const __nv_bfloat16* bias, const HeadOut out,
                           int n_valid, int K, int kb_split, int rows, const HeadStd sd, const HeadEps eg,
                           const HeadEval ev, const HeadQ hq) {
  const int n0 = blockIdx.x * BLOCK_N;
  const int m0 = blockIdx.y * kMlpBlockM;
  const int lane = threadIdx.x & 31;
  const int col0 = n0 + 2 * (lane & 3);
  float acc[BLOCK_N / 2];
  if (!mlp_tile_mainloop<BLOCK_N, STAGES>(maps_a.m, &map_b, K, kb_split, m0, n0, acc)) return;
  const int warp = threadIdx.x >> 5;
  const int wg = warp >> 2;

  // accumulator layout of m64nNk16: acc[4j + 2h + c] is row 16*(warp%4) + lane/4 + 8h, column 8j + 2*(lane%4) + c
  const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const bool st0 = row < rows, st1 = row + 8 < rows;
  __nv_bfloat16* C = static_cast<__nv_bfloat16*>(out.logits);
  if constexpr (KIND == HeadKind::kHidden) {
    store_tile<BLOCK_N, true>(acc, bias, C, col0, n_valid, row, st0, st1);
  } else if constexpr (KIND == HeadKind::kGreedy) {
    greedy_epilogue<BLOCK_N>(acc, bias, C, out.actions, out.mask, col0, n_valid, row, st0, st1);
  } else if constexpr (KIND == HeadKind::kSample) {
    sample_epilogue<BLOCK_N, STAGES>(acc, bias, col0, n_valid, row, st0, st1, out.actions, out.log_probs, out.mask, out.seed,
                             out.row_base, out.values, out.groups, C, eg.epsilon, eg.q, eg.q_max, ev, hq);
  } else if (BLOCK_N == 64 && (hq.q != nullptr || hq.y != nullptr)) {   // a critic (64-wide tile): column 0 is Q
    critic_epilogue<BLOCK_N>(acc, bias, col0, row, st0, st1, hq);
  } else {
    gaussian_epilogue<BLOCK_N, STAGES>(acc, bias, col0, n_valid, row, st0, st1, out.log_std, out.gauss_actions,
                                       out.log_probs, out.seed, out.row_base, out.values, sd, ev);
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

// One layer through the epilogue of KIND in BLOCK_N-wide tiles: out = A[M, K] · B[N, K]ᵀ (+ bias), N columns.  With
// `tile` (a critic's layer 1) A is [M, K − 64] and its last K block is tile [M, 64] instead.
template <int BLOCK_N, HeadKind KIND>
static int launch_layer(int dev, const void* A, const void* B, const void* bias, const HeadOut& out, size_t M, int N,
                        int K, cudaStream_t stream, const HeadStd& sd = HeadStd{}, const HeadEps& eg = HeadEps{},
                        const HeadEval& ev = HeadEval{}, const HeadQ& hq = HeadQ{}, const void* tile = nullptr) {
  using S = MlpSmem<BLOCK_N, kMlpStages>;
  static_assert(S::kTotal <= 232448, "the TMA ring must fit the 227 KiB a block may own");
  const int k_a = tile ? K - kMlpBlockK : K;   // A's own columns
  CUtensorMap mb;
  AMaps am;
  CUtensorMap& ma = am.m[0];
  CUtensorMap& ma2 = am.m[1];
  int rc = make_map(&ma, A, M, (uint64_t)k_a, kMlpBlockM);
  if (rc) return rc;
  rc = make_map(&mb, B, (uint64_t)N, (uint64_t)K, BLOCK_N);
  if (rc) return rc;
  ma2 = ma;
  if (tile) {
    rc = make_map(&ma2, tile, M, kMlpBlockK, kMlpBlockM);
    if (rc) return rc;
  }
  auto kfn = mlp_layer_wgmma_kernel<BLOCK_N, kMlpStages, KIND>;
  static std::atomic<unsigned> attr_done{0};
  rc = ensure_smem_attr(kfn, S::kTotal, attr_done, dev);
  if (rc) return rc;
  dim3 grid((unsigned)((N + BLOCK_N - 1) / BLOCK_N), (unsigned)((M + kMlpBlockM - 1) / kMlpBlockM));
  kfn<<<grid, kMlpThreads, S::kTotal, stream>>>(am, mb, static_cast<const __nv_bfloat16*>(bias), out, N, K,
                                                k_a / kMlpBlockK, (int)M, sd, eg, ev, hq);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

// The head of KIND, in the smallest tile that holds its N columns (d_out, 2·d_out for a state-dependent Gaussian
// head, one more with a value head).
template <HeadKind KIND>
static int launch_head(int dev, const void* A, const void* B, const void* bias, const HeadOut& out, size_t M, int N,
                       int K, cudaStream_t stream, const HeadStd& sd, const HeadEps& eg, const HeadEval& ev,
                       const HeadQ& hq) {
  const auto launch = N <= 64 ? launch_layer<64, KIND> : N <= 128 ? launch_layer<128, KIND> : launch_layer<256, KIND>;
  return launch(dev, A, B, bias, out, M, N, K, stream, sd, eg, ev, hq, nullptr);
}

// A critic's action tile: tile[r, j] = bf16(act[r, j]) (round to nearest even, as torch's .to(torch.bfloat16)) for
// j < d_act and 0 for d_act <= j < 64, over `rows` rows of fp32 act [rows, d_act] (4-byte aligned; may be a peer
// pointer).  One thread per 8 columns of a row, one 16-byte store.
__global__ void critic_action_tile_kernel(const float* act, int d_act, __nv_bfloat16* tile, size_t rows) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= rows * 8) return;
  const size_t r = t >> 3;
  const int c0 = (int)(t & 7) * 8;
  const float* a = act + r * d_act;
  __align__(16) __nv_bfloat16 v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = __float2bfloat16_rn(c0 + c < d_act ? a[c0 + c] : 0.f);
  *reinterpret_cast<uint4*>(tile + r * kMlpBlockK + c0) = *reinterpret_cast<const uint4*>(v);
}

static int launch_action_tile(const float* act, int d_act, void* tile, size_t rows, cudaStream_t st) {
  const size_t threads = rows * 8;
  critic_action_tile_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(act, d_act,
                                                                              static_cast<__nv_bfloat16*>(tile), rows);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

// Weights and biases (each bias may be null) of one MLP call, and its head.  `logits64` marks ktb_mlp_bf16, _staged and
// _pushed: no biases and a 64-wide greedy head that stores logits only.  `masked` marks the _masked entries: the head
// applies a legal-action mask, out.mask in the pull forms and the call's "mask" side (MlpFeed) in the pushed forms.
// `valued` marks the _value entries: W3 / b3 are the stacked W3v [d_out + 1, d_hidden] / b3v [d_out + 1] of the policy
// and its value head, and out.values receives the value of each row. `nvec` (n_groups entries, a host array) marks the
// _multidiscrete entries: mlp_run checks it and builds out.groups. std.state marks the _gaussian_state entries: W3 / b3
// are the interleaved W3s [2·d_out, d_hidden] / b3s (with a value head W3sv / b3sv, one more row), log_std is null, and
// mlp_run checks the bounds.  `eps` marks the _epsilon_greedy entries: eg.epsilon (the pull forms) or the call's
// "epsilon" side (the pushed forms) hold each row's ε, and out.actions, eg.q and eg.q_max receive the outputs.
// `evaluate` marks the _evaluate entries: ev.actions (kSample) or ev.gauss_actions (kGaussian), or in the pushed forms
// the call's "taken" side, hold the given actions, and out.log_probs and ev.entropy receive the outputs; a categorical
// one is grouped unless nvec == null and n_groups == 0.  std.det marks the _deterministic entries: out.gauss_actions
// receives the actions, and mlp_run checks σ and the clip.  `critic` marks the _critic entries: W1 is W1p [d_hidden,
// d_in + 64], layer 1 reads an action tile packed from `act` (fp32 [M, d_act]; in the pushed forms the call's "act"
// side) as its last K block, W3 / b3 are the critic's [1, d_hidden] / [1], and hq receives Q; `twin` (the _twin
// entries) is the second critic, run on the same tile after the first, whose hq also reads the first's q and stores
// q_min.  `actor` marks the _td_target entries: the critics' action tile is packed from the actions the actor (a
// deterministic or state-dependent Gaussian head, `actor_hidden` wide) writes into chunk scratch, and the last critic's
// hq computes the target (`target` marks both critics: their hq reads and writes chunk scratch).  `dqn` marks the
// _dqn_target entries: a kSample head whose hq computes the target from the target network's logits (`target` set too),
// at the actions that `online` (Double DQN; a greedy head, masked with the call's mask) writes into chunk scratch, or
// without `online` at its own greedy actions under the call's mask.
struct MlpParams {
  const void *W1, *b1, *W2, *b2, *W3, *b3;
  HeadKind kind;
  HeadOut out;
  bool logits64 = false;
  bool masked = false;
  bool valued = false;
  const int32_t* nvec = nullptr;
  int n_groups = 0;
  bool grouped = false;
  HeadStd std;
  bool eps = false;
  HeadEps eg;
  bool evaluate = false;
  HeadEval ev;
  bool critic = false;
  int d_act = 0;
  const float* act = nullptr;
  HeadQ hq;
  const MlpParams* twin = nullptr;
  const MlpParams* actor = nullptr;
  int actor_hidden = 0;
  bool target = false;
  bool dqn = false;
  const MlpParams* online = nullptr;

  // A critic, in the 64-wide kGaussian instantiation (one column, Q): act [M, d_act] fp32 (null in the pushed forms)
  // in, q [M] fp32 out.
  static MlpParams critic_head(const void* W1p, const void* b1, const void* W2, const void* b2, const void* W3,
                               const void* b3, int d_act, const float* act, float* q) {
    MlpParams p{W1p, b1, W2, b2, W3, b3, HeadKind::kGaussian};
    p.critic = true;
    p.d_act = d_act;
    p.act = act;
    p.hq = HeadQ{q};
    return p;
  }

  // A multi-discrete head: the greedy one (logits and/or actions, ranked without noise) or the sampled one, both in
  // the kSample instantiations.
  static MlpParams multidiscrete(const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                 const void* b3, const int32_t* nvec, int n_groups, const HeadOut& out, bool greedy) {
    MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kSample, out};
    p.out.groups.greedy = greedy;
    p.nvec = nvec;
    p.n_groups = n_groups;
    p.grouped = true;
    return p;
  }

  // A state-dependent Gaussian head, in the kGaussian instantiations: log-std bounds [lo, hi], tanh with squash != 0.
  static MlpParams gaussian_state(const void* W1, const void* b1, const void* W2, const void* b2, const void* W3s,
                                  const void* b3s, float lo, float hi, int squash, const HeadOut& out) {
    MlpParams p{W1, b1, W2, b2, W3s, b3s, HeadKind::kGaussian, out};
    p.std = HeadStd{lo, hi, true, squash != 0};
    return p;
  }

  // An ε-greedy head, in the kSample instantiations: epsilon [M] in (null in the pushed forms), actions, q, q_max out.
  static MlpParams epsilon_greedy(const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                  const void* b3, const float* epsilon, uint64_t seed, uint64_t row_base,
                                  int64_t* actions, float* q, float* q_max) {
    MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, actions, nullptr, seed, row_base}};
    p.eg = HeadEps{epsilon, q, q_max};
    p.eps = true;
    return p;
  }

  // A categorical evaluating head, in the kSample instantiations: taken [M] or [M, n_groups] int64 (null in the pushed
  // forms) in, log_probs and entropy out.  nvec == null with n_groups == 0 is the single categorical.
  static MlpParams evaluate_categorical(const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                        const void* b3, const int32_t* nvec, int n_groups, const int64_t* taken,
                                        float* log_probs, float* entropy) {
    MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, nullptr, log_probs}};
    p.grouped = nvec != nullptr || n_groups != 0;
    p.nvec = nvec;
    p.n_groups = n_groups;
    p.evaluate = true;
    p.ev = HeadEval{taken, nullptr, entropy};
    return p;
  }

  // A deterministic actor, in the kGaussian instantiations: actions [M, d_out] fp32 out, σ = noise, clip, tanh with
  // squash != 0.
  static MlpParams deterministic(const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                 const void* b3, float noise, float clip, int squash, uint64_t seed, uint64_t row_base,
                                 float* actions) {
    MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGaussian, {nullptr, nullptr, nullptr, seed, row_base, nullptr, actions}};
    p.std.det = true;
    p.std.squash = squash != 0;
    p.std.noise = noise;
    p.std.clip = clip;
    return p;
  }

  // A state-independent Gaussian evaluating head, in the kGaussian instantiations: taken [M, d_out] fp32 (null in the
  // pushed forms) in, log_probs and entropy out.
  static MlpParams evaluate_gaussian(const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                     const void* b3, const float* log_std, const float* taken, float* log_probs,
                                     float* entropy) {
    MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGaussian, {nullptr, nullptr, log_probs, 0, 0, log_std}};
    p.evaluate = true;
    p.ev = HeadEval{nullptr, taken, entropy};
    return p;
  }

  MlpParams with_mask(const uint8_t* mask) const {
    MlpParams p = *this;
    p.out.mask = mask;
    p.masked = true;
    return p;
  }
  MlpParams with_values(float* values) const {
    MlpParams p = *this;
    p.out.values = values;
    p.valued = true;
    return p;
  }
};

// Rows [r0, r0 + rows) of a call: the hidden layers h1 = relu(a1 · W1ᵀ (+ b1)) and h2 = relu(h1 · W2ᵀ (+ b2)), then
// the head of p.kind into `out` (the call's outputs, from row 0) from h2 in the smallest tile that holds its d_out
// columns (2·d_out for a state-dependent Gaussian head), one more with a value head.  A critic's layer 1 reads
// `tile` (the chunk's actions) as its last K block.  `consumed`, unless null, is recorded once layer 1 has read a1.
static int mlp_chunk(int dev, const MlpParams& p, const HeadOut& out, const HeadEps& eg, const HeadEval& ev,
                     const void* a1, const void* tile, void* h1, void* h2, size_t r0, size_t rows, int d_in,
                     int d_hidden, int d_out, cudaEvent_t consumed, cudaStream_t st) {
  int rc = launch_layer<256, HeadKind::kHidden>(dev, a1, p.W1, p.b1, HeadOut{h1}, rows, d_hidden,
                                                d_in + (p.critic ? kMlpBlockK : 0), st, HeadStd{}, HeadEps{},
                                                HeadEval{}, HeadQ{}, p.critic ? tile : nullptr);
  if (rc) return rc;
  if (consumed) KTB_CK(cudaEventRecord(consumed, st));
  rc = launch_layer<256, HeadKind::kHidden>(dev, h1, p.W2, p.b2, HeadOut{h2}, rows, d_hidden, d_hidden, st);
  if (rc) return rc;
  const auto head = p.kind == HeadKind::kGreedy   ? launch_head<HeadKind::kGreedy>
                    : p.kind == HeadKind::kSample ? launch_head<HeadKind::kSample>
                                                  : launch_head<HeadKind::kGaussian>;
  const int n = (p.std.state ? 2 * d_out : d_out) + (int)p.valued;
  const size_t per_row = ev.gauss_actions ? (size_t)d_out : (size_t)std::max(out.groups.n, 1);   // given actions
  return head(dev, h2, p.W3, p.b3, out.from_row(r0, d_out), rows, n, d_hidden, st, p.std, eg.from_row(r0),
              ev.from_row(r0, per_row), p.hq.from_row(r0, p.target));
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
      case HeadKind::kHidden:   // the hidden layers' epilogue, never an entry point's head
        break;
      case HeadKind::kGreedy:
        KTB_REQUIRE(o.logits || o.actions, KTB_ERR_ARG, "%s: logits and actions are both null", fn);
        break;
      case HeadKind::kSample:
        if (o.groups.greedy)   // a greedy multi-discrete head takes what the greedy entries take
          KTB_REQUIRE(o.logits || o.actions, KTB_ERR_ARG, "%s: logits and actions are both null", fn);
        else if (!p.eps && !p.evaluate && !p.dqn)   // ε-greedy, evaluating and DQN target heads: checked by mlp_run
          KTB_REQUIRE(o.actions && o.log_probs, KTB_ERR_ARG, "%s: actions and log_probs are required", fn);
        break;
      case HeadKind::kGaussian:
        if (p.critic)   // a critic's act and outputs: checked by mlp_run after every other check
          break;
        if (p.std.det)   // a deterministic actor stores its actions only
          KTB_REQUIRE(o.gauss_actions, KTB_ERR_ARG, "%s: actions is required", fn);
        else if (p.std.state)   // a state-dependent head reads its log-std from the head's own columns
          KTB_REQUIRE(o.gauss_actions && o.log_probs, KTB_ERR_ARG, "%s: actions and log_probs are required", fn);
        else if (p.evaluate)   // an evaluating head's actions and outputs are checked by mlp_run after every other check
          KTB_REQUIRE(o.log_std, KTB_ERR_ARG, "%s: log_std is required", fn);
        else
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

// How the rows of each chunk of a call reach layer 1: the form of an entry point.
//   plain : layer 1 reads the chunk in `in` (obs).
//   staged: (stage != null) the chunk is pulled from `in` (obs on a peer) into half c & 1 of `stage` on the device's
//           stage stream while the previous chunk computes, and layer 1 reads it there.
//   pushed: the root pushes the rows into half seq & 1 of `in` (stage_local, halves `stride` bytes apart) and publishes
//           ready[c] = seq in this rank's control block `ctrl`; layer 1 of chunk c waits in-stream for it, and the
//           call ends by publishing ack[rank] = seq in the root's control block `ctrl_root`.  A head's per-row
//           inputs were pushed into the same half beside the rows: `sides`, up to two regions (PushSide, src null)
//           named for what they hold, "mask" (a masked head's legal-action mask), "epsilon" (an ε-greedy head's ε,
//           fp32), "taken" (an evaluating head's given actions), "act" (a critic's actions, fp32), or "reward" and
//           "done" (a TD target's, fp32), or "rd" (a DQN target's interleaved fp32 (reward, done) pairs).
// The pull forms read a mask in place (MlpParams::out.mask), a peer pointer where obs is one: it is read once per row.
struct MlpFeed {
  const void* in;
  size_t chunk_rows;
  void* stage = nullptr;
  bool pushed = false;
  size_t stride = 0;
  void *ctrl = nullptr, *ctrl_root = nullptr;
  int rank = 0;
  unsigned long long seq = 0;
  PushSide sides[2] = {};
  int n_sides = 0;

  static MlpFeed pull(const void* obs, void* stage) { return {obs, (size_t)g_mlp_chunk_rows, stage}; }
  static MlpFeed push(const void* stage_local, size_t stride, void* ctrl, void* ctrl_root, int rank, size_t chunk_rows,
                      unsigned long long seq) {
    return {stage_local, chunk_rows, nullptr, true, stride, ctrl, ctrl_root, rank, seq};
  }
  // the feed with one more side region: `name`, `offset` bytes into the half, row_bytes per row, `align`-aligned
  MlpFeed with_side(const char* name, size_t offset, size_t row_bytes, size_t align) const {
    MlpFeed f = *this;
    f.sides[f.n_sides++] = PushSide{nullptr, row_bytes, offset, align, name};
    return f;
  }
  // the side named `name` in staging half `half`
  const void* side(const uint8_t* half, const char* name) const {
    for (int k = 0; k < n_sides; ++k)
      if (strcmp(sides[k].name, name) == 0) return half + sides[k].offset;
    return nullptr;
  }
};

// The chunk scratch of a call, in this order: two hidden activations [chunk, d_hidden] bf16 (a TD target's actor and
// critics share them, at the wider d_hidden, and a DQN target's two networks), a critic's action tile [chunk, 64] bf16,
// then a TD target's actions [chunk, d_act], log-probabilities [chunk] and first Q [chunk], fp32
// (ktb_mlp_td_target_scratch_bytes).  A DQN target's selected actions [chunk] int64 take the place of the action tile
// (ktb_mlp_dqn_target_scratch_bytes).
struct MlpScratch {
  __nv_bfloat16 *h1, *h2, *tile;
  float *act, *logp, *q1;
  int64_t* sel;

  static MlpScratch carve(void* scratch, size_t chunk, int d_hidden, int d_act) {
    MlpScratch s;
    s.h1 = static_cast<__nv_bfloat16*>(scratch);
    s.h2 = s.h1 + chunk * (size_t)d_hidden;
    s.tile = s.h2 + chunk * (size_t)d_hidden;
    s.act = reinterpret_cast<float*>(s.tile + chunk * (size_t)kMlpBlockK);
    s.logp = s.act + chunk * (size_t)d_act;
    s.q1 = s.logp + chunk;
    s.sel = reinterpret_cast<int64_t*>(s.tile);
    return s;
  }
};

// The checks of a head's own options, skipped for an empty call: a value head's values and width, a state-dependent
// Gaussian head's width and log-std bounds, a deterministic actor's noise and noise_clip.
static int head_checks(const char* fn, size_t M, int d_out, const MlpParams& p) {
  if (p.valued && M > 0) {
    KTB_REQUIRE(p.out.values, KTB_ERR_ARG, "%s: null values", fn);
    KTB_REQUIRE(((uintptr_t)p.out.values & 3) == 0, KTB_ERR_ARG, "%s: values must be 4-byte aligned", fn);
    KTB_REQUIRE(d_out <= 255, KTB_ERR_UNSUPPORTED, "%s: d_out=%d (the policy and its value column fit one 256-wide tile)",
                fn, d_out);
  }
  if (p.std.state && M > 0) {
    KTB_REQUIRE(2 * d_out + (int)p.valued <= 256, KTB_ERR_UNSUPPORTED,
                "%s: d_out=%d (the interleaved mean and log-std%s fit one 256-wide tile)", fn, d_out,
                p.valued ? " and the value column" : "");
    const float lo = p.std.lo, hi = p.std.hi;
    KTB_REQUIRE(lo == lo && hi == hi && lo <= hi, KTB_ERR_ARG, "%s: log_std bounds [%g, %g] must be ordered, not NaN",
                fn, (double)lo, (double)hi);
  }
  if (p.std.det && M > 0) {
    const float s = p.std.noise, c = p.std.clip;
    KTB_REQUIRE(s == s && s >= 0.f, KTB_ERR_ARG, "%s: noise=%g must be >= 0, not NaN", fn, (double)s);
    KTB_REQUIRE(c == c && c >= 0.f, KTB_ERR_ARG, "%s: noise_clip=%g must be >= 0, not NaN", fn, (double)c);
  }
  return KTB_OK;
}

// The weights and biases of a second network of the same shapes (a twin's second critic, a Double DQN target's online
// network): non-null weights, and the alignment mlp_check asks of the first's.
static int second_network_check(const char* fn, size_t M, const MlpParams& t) {
  KTB_REQUIRE(t.W1 && t.W2 && t.W3, KTB_ERR_ARG, "%s: null argument", fn);
  KTB_REQUIRE(M == 0 || (((uintptr_t)t.b1 | (uintptr_t)t.b2 | (uintptr_t)t.b3) & 1) == 0, KTB_ERR_ARG,
              "%s: logits and biases must be 2-byte aligned", fn);
  KTB_REQUIRE((((uintptr_t)t.W1 | (uintptr_t)t.W2 | (uintptr_t)t.W3) & 15) == 0, KTB_ERR_ARG,
              "%s: obs, weights, scratch and stage must be 16-byte aligned", fn);
  return KTB_OK;
}

// One MLP call of any head and form: every entry's checks, then one chunk loop.  An empty plain or staged call returns
// right after the device check; an empty pushed shard runs every check and still publishes its ack, which the root's
// ktb_push_wait waits for.  A pushed entry's side regions (check_push_sides) are checked right after its stage_stride,
// before every check of the head's own arguments, so a call with a bad region and another defect may report the
// region's KTB_ERR_ARG first.  A masked entry's own checks (a mask in the pull forms) come after every check of the
// unmasked entry, and a value entry's (values, d_out <= 255; skipped for an empty call) after every check of the entry
// without a value head.  A multi-discrete entry's nvec (skipped for an empty call) is checked last, and read into the
// launch's HeadGroups before the call returns.  A state-dependent Gaussian entry's head width (2·d_out, one more with a
// value head, <= 256) and log-std bounds (skipped for an empty call) come after every check of its state-independent
// counterpart.  An ε-greedy entry's own checks come after every check of its greedy counterpart (ktb_mlp_bf16_policy or
// _masked): (skipped for an empty call) ε, actions, q and q_max non-null and aligned.  An evaluating entry's own checks
// come after every check of its counterpart and its nvec: (skipped for an empty call) taken, log_probs, entropy
// non-null and aligned.  A deterministic entry's actions are checked with the head (mlp_check), its noise and
// noise_clip (>= 0, not NaN; skipped for an empty call) after every check.  A critic entry runs every check of
// ktb_mlp_bf16_policy at d_out = 1 (a twin's second critic's weights and biases checked as the first's, right after
// them), then d_act in [1, 64], then (skipped for an empty call) act and its outputs non-null and 4-byte aligned.  A TD
// target entry runs every check of the critic (twin) entry but those of act and the Q outputs, then every check of its
// actor's standalone entry (ktb_mlp_bf16_policy_deterministic or _gaussian_state at d_out = d_act, the actor's
// d_hidden), then gamma and alpha finite, then (skipped for an empty call) reward, done and y non-null and aligned.  A
// DQN target entry runs every check of ktb_mlp_bf16_policy (_masked) on the target network, then the online network's
// as a twin's second critic's, then gamma finite, then (skipped for an empty call) reward, done and y non-null and
// aligned.
static int mlp_run(const char* fn, int dev, size_t M, int d_in, int d_hidden, int d_out, const MlpParams& p,
                   const MlpFeed& f, void* scratch, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  if (M == 0 && !f.pushed) return KTB_OK;
  if (p.logits64) {
    KTB_REQUIRE(p.out.logits || M == 0, KTB_ERR_ARG, "%s: null argument", fn);
    KTB_REQUIRE(d_out == 64, KTB_ERR_UNSUPPORTED, "%s: d_out=%d (the 64-wide head)", fn, d_out);
    KTB_REQUIRE(f.pushed || ((uintptr_t)p.out.logits & 15) == 0, KTB_ERR_ARG, "%s: logits must be 16-byte aligned",
                fn);
  }
  KTB_REQUIRE(f.in && p.W1 && p.W2 && p.W3 && scratch && (!f.pushed || (f.ctrl && f.ctrl_root)), KTB_ERR_ARG,
              "%s: null argument", fn);
  if (f.pushed) {
    KTB_REQUIRE(f.rank >= 0 && f.rank < 16 && f.seq > 0, KTB_ERR_ARG, "%s: bad rank/seq", fn);
    KTB_REQUIRE(M % kMlpBlockM == 0, KTB_ERR_ARG, "%s: M=%zu must be a multiple of %d", fn, M, kMlpBlockM);
  }
  KTB_REQUIRE(f.chunk_rows > 0 && f.chunk_rows % kMlpBlockM == 0, KTB_ERR_ARG,
              "%s: chunk_rows=%zu must be a positive multiple of %d", fn, f.chunk_rows, kMlpBlockM);
  rc = mlp_check(fn, M, d_in, d_hidden, d_out, p, f.in, scratch, f.stage);
  if (rc) return rc;
  if (p.twin) {
    rc = second_network_check(fn, M, *p.twin);
    if (rc) return rc;
  }
  if (f.pushed) {
    const size_t n_chunks = (M + f.chunk_rows - 1) / f.chunk_rows;
    KTB_REQUIRE(n_chunks <= KTB_PUSH_MAX_CHUNKS, KTB_ERR_ARG, "%s: %zu chunks exceed %d", fn, n_chunks,
                KTB_PUSH_MAX_CHUNKS);
    KTB_REQUIRE(M * (size_t)d_in * 2 <= f.stride, KTB_ERR_ARG, "%s: shard exceeds stage_stride", fn);
    // layer 1 reads half seq & 1 through a tensor map, whose base TMA needs 16-byte aligned
    KTB_REQUIRE(f.stride % 16 == 0, KTB_ERR_ARG, "%s: stage_stride=%zu must be a multiple of 16", fn, f.stride);
    rc = check_push_sides(fn, f.sides, f.n_sides, M, (size_t)d_in * 2, f.stride);
    if (rc) return rc;
  }
  if (p.masked && !f.pushed)
    KTB_REQUIRE(p.out.mask, KTB_ERR_ARG, "%s: null mask", fn);   // M > 0 here: an empty pull call has returned
  if (p.eps && M > 0) {
    const HeadEps& o = p.eg;
    KTB_REQUIRE((o.epsilon || f.pushed) && p.out.actions && o.q && o.q_max, KTB_ERR_ARG,
                "%s: epsilon, actions, q and q_max are required", fn);
    KTB_REQUIRE((((uintptr_t)o.epsilon | (uintptr_t)o.q | (uintptr_t)o.q_max) & 3) == 0, KTB_ERR_ARG,
                "%s: epsilon, q and q_max must be 4-byte aligned", fn);
  }
  rc = head_checks(fn, M, d_out, p);
  if (rc) return rc;
  if (p.critic) {
    KTB_REQUIRE(p.d_act >= 1, KTB_ERR_ARG, "%s: d_act=%d must be positive", fn, p.d_act);
    KTB_REQUIRE(p.d_act <= kMlpBlockK, KTB_ERR_UNSUPPORTED, "%s: d_act=%d (actions up to %d wide)", fn, p.d_act,
                kMlpBlockK);
    if (M > 0 && !p.actor) {
      const HeadQ& q2 = p.twin ? p.twin->hq : HeadQ{};
      KTB_REQUIRE((p.act || f.pushed) && p.hq.q && (!p.twin || (q2.q && q2.q_min)), KTB_ERR_ARG,
                  p.twin ? "%s: act, q1, q2 and q_min are required" : "%s: act and q are required", fn);
      KTB_REQUIRE((((uintptr_t)p.act | (uintptr_t)p.hq.q | (uintptr_t)q2.q | (uintptr_t)q2.q_min) & 3) == 0,
                  KTB_ERR_ARG, "%s: act and the outputs must be 4-byte aligned", fn);
    }
  }
  if (p.dqn) {
    if (p.online) {
      rc = second_network_check(fn, M, *p.online);
      if (rc) return rc;
    }
    const HeadQ& t = p.hq;
    KTB_REQUIRE(std::isfinite(t.gamma), KTB_ERR_ARG, "%s: gamma=%g must be finite", fn, (double)t.gamma);
    if (M > 0) {
      KTB_REQUIRE(((t.reward && t.done) || f.pushed) && t.y, KTB_ERR_ARG, "%s: reward, done and y are required", fn);
      KTB_REQUIRE((((uintptr_t)t.reward | (uintptr_t)t.done | (uintptr_t)t.y) & 3) == 0, KTB_ERR_ARG,
                  "%s: reward, done and y must be 4-byte aligned", fn);
    }
  }
  const size_t chunk = std::min(f.chunk_rows, M);
  const MlpScratch s = MlpScratch::carve(scratch, chunk, std::max(d_hidden, p.actor_hidden), p.d_act);
  // a TD target's actor and critics with their chunk scratch: the actor writes its actions (and log-probabilities)
  // there, the first of two critics its Q, and the last critic reads them
  MlpParams actor{}, c1 = p, c2{};
  if (p.actor) {
    actor = *p.actor;
    actor.out.gauss_actions = s.act;
    if (actor.std.state) actor.out.log_probs = s.logp;
    KTB_REQUIRE(actor.W1 && actor.W2 && actor.W3, KTB_ERR_ARG, "%s: null argument", fn);
    rc = mlp_check(fn, M, d_in, p.actor_hidden, p.d_act, actor, f.in, scratch, f.stage);
    if (rc) return rc;
    rc = head_checks(fn, M, p.d_act, actor);
    if (rc) return rc;
    if (p.twin) {
      c2 = *p.twin;
      c1.hq.q = s.q1;
      c2.hq.q_other = s.q1;
      c1.twin = &c2;
    }
    HeadQ& t = (p.twin ? c2 : c1).hq;
    KTB_REQUIRE(std::isfinite(t.gamma) && std::isfinite(t.alpha), KTB_ERR_ARG, "%s: gamma=%g and alpha=%g must be finite",
                fn, (double)t.gamma, (double)t.alpha);
    if (M > 0) {
      KTB_REQUIRE(((t.reward && t.done) || f.pushed) && t.y, KTB_ERR_ARG, "%s: reward, done and y are required", fn);
      KTB_REQUIRE((((uintptr_t)t.reward | (uintptr_t)t.done | (uintptr_t)t.y) & 3) == 0, KTB_ERR_ARG,
                  "%s: reward, done and y must be 4-byte aligned", fn);
    }
    if (actor.std.state) t.logp = s.logp;
  }
  // a Double DQN target's online network writes the chunk's actions into chunk scratch, where the target's head reads
  // them
  MlpParams online{};
  if (p.online) {
    online = *p.online;
    online.out.actions = s.sel;
    c1.hq.sel = s.sel;
  }
  HeadGroups groups = p.out.groups;
  if (p.grouped && M > 0) {
    KTB_REQUIRE(p.nvec, KTB_ERR_ARG, "%s: null nvec", fn);
    KTB_REQUIRE(p.n_groups >= 1 && p.n_groups <= d_out, KTB_ERR_ARG, "%s: n_groups=%d must be in [1, d_out=%d]", fn,
                p.n_groups, d_out);
    long long lo = 0;
    for (int g = 0; g < p.n_groups; ++g) {
      KTB_REQUIRE(p.nvec[g] >= 1, KTB_ERR_ARG, "%s: nvec[%d]=%d must be positive", fn, g, (int)p.nvec[g]);
      if (lo < d_out) groups.starts[lo >> 5] |= 1u << (lo & 31);
      lo += p.nvec[g];
    }
    KTB_REQUIRE(lo == d_out, KTB_ERR_ARG, "%s: nvec sums to %lld, not d_out=%d", fn, lo, d_out);
    groups.n = p.n_groups;
  }
  if (p.evaluate) {
    const bool cat = p.kind == HeadKind::kSample;
    const void* taken = cat ? (const void*)p.ev.actions : (const void*)p.ev.gauss_actions;
    const size_t align = cat ? 8 : 4;
    if (M > 0) {
      KTB_REQUIRE((taken || f.pushed) && p.out.log_probs && p.ev.entropy, KTB_ERR_ARG,
                  "%s: taken, log_probs and entropy are required", fn);
      KTB_REQUIRE((uintptr_t)taken % align == 0, KTB_ERR_ARG, "%s: taken must be %zu-byte aligned", fn, align);
      KTB_REQUIRE((((uintptr_t)p.out.log_probs | (uintptr_t)p.ev.entropy) & 3) == 0, KTB_ERR_ARG,
                  "%s: log_probs and entropy must be 4-byte aligned", fn);
    }
  }
  rc = get_encoder();
  if (rc) return rc;
  KTB_GUARD(dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the call's rows: obs, or this call's staging half (the pull forms have seq = stride = 0)
  const uint8_t* half = static_cast<const uint8_t*>(f.in) + (size_t)(f.seq & 1) * f.stride;
  const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(half);
  HeadOut out = p.out;
  out.groups = groups;
  HeadEps eg = p.eg;
  HeadEval ev = p.ev;
  const float* act = p.act;
  if (f.pushed) {   // the head's per-row inputs, pushed into the same half
    if (p.masked) out.mask = static_cast<const uint8_t*>(f.side(half, "mask"));
    if (p.eps) eg.epsilon = static_cast<const float*>(f.side(half, "epsilon"));
    if (p.evaluate && p.kind == HeadKind::kSample) ev.actions = static_cast<const int64_t*>(f.side(half, "taken"));
    if (p.evaluate && p.kind != HeadKind::kSample) ev.gauss_actions = static_cast<const float*>(f.side(half, "taken"));
    if (p.critic && !p.actor) act = static_cast<const float*>(f.side(half, "act"));
    if (p.actor) {
      HeadQ& t = (p.twin ? c2 : c1).hq;
      t.reward = static_cast<const float*>(f.side(half, "reward"));
      t.done = static_cast<const float*>(f.side(half, "done"));
    }
    if (p.dqn) {   // interleaved (reward, done) pairs
      c1.hq.reward = static_cast<const float*>(f.side(half, "rd"));
      c1.hq.done = c1.hq.reward + 1;
      c1.hq.rd_stride = 2;
    }
  }
  // Double DQN masks the online network's ranking; the target's value is read unmasked
  const uint8_t* online_mask = out.mask;
  if (p.online) out.mask = nullptr;
  uint8_t* ctrl = static_cast<uint8_t*>(f.ctrl);
  __nv_bfloat16* stg = static_cast<__nv_bfloat16*>(f.stage);
  cudaStream_t side = device_info(dev)->stream_stage;   // pulls the next chunk while this one computes
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
  static std::mutex side_mu[kMaxDevices];   // the stage stream of a device carries one staged call at a time
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
    if (f.pushed) {
      // one warp spins until the root's ready[c] = seq (a timeout raises the sticky status)
      rc = launch_flag_wait(reinterpret_cast<const unsigned long long*>(ctrl + KTB_CTRL_READY) + c, f.seq,
                            reinterpret_cast<unsigned int*>(ctrl + KTB_CTRL_STATUS), st);
      if (rc) return rc;
    } else if (stg) {
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
    // evs[3..4] are null unless staged; every chain after the first records `consumed` again after its layer 1
    cudaEvent_t consumed = evs[3 + (int)(c & 1)];
    if (p.online) {   // the chunk's greedy actions into chunk scratch: pointers from its row 0
      HeadOut so = online.out;
      so.mask = online_mask ? online_mask + r0 * d_out : nullptr;
      rc = mlp_chunk(dev, online, so, HeadEps{}, HeadEval{}, a1, nullptr, s.h1, s.h2, 0, rows, d_in, d_hidden, d_out,
                     consumed, st);
      if (rc) return rc;
    }
    if (p.actor) {   // the chunk's actions into chunk scratch: pointers from its row 0, noise of its global rows
      HeadOut ao = actor.out;
      ao.row_base += r0;
      rc = mlp_chunk(dev, actor, ao, HeadEps{}, HeadEval{}, a1, nullptr, s.h1, s.h2, 0, rows, d_in, p.actor_hidden,
                     p.d_act, consumed, st);
      if (rc) return rc;
    }
    if (p.critic) {   // packed once per chunk; a twin's two chains both read it
      rc = launch_action_tile(p.actor ? s.act : act + r0 * p.d_act, p.d_act, s.tile, rows, st);
      if (rc) return rc;
    }
    for (const MlpParams* q = &c1; q != nullptr; q = q->twin) {
      rc = mlp_chunk(dev, *q, out, eg, ev, a1, s.tile, s.h1, s.h2, r0, rows, d_in, d_hidden, d_out, consumed, st);
      if (rc) return rc;
    }
  }
  if (!f.pushed) return KTB_OK;
  // everything before it on `st`, the peer-stored outputs included, is visible system-wide before the root sees
  // ack[rank] = seq
  return launch_flag_publish(
      reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(f.ctrl_root) + KTB_CTRL_ACK) + f.rank, f.seq, st);
}
}  // namespace ktb

using namespace ktb;

extern "C" {

size_t ktb_mlp_scratch_bytes(size_t M, int d_hidden) {
  const size_t rows = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  return 2 * rows * (size_t)d_hidden * 2;
}

size_t ktb_mlp_critic_scratch_bytes(size_t M, int d_hidden) {
  const size_t rows = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  return ktb_mlp_scratch_bytes(M, d_hidden) + rows * (size_t)kMlpBlockK * 2;
}

size_t ktb_mlp_stage_bytes(size_t M, int d_in) {
  const size_t rows = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  return 2 * rows * (size_t)d_in * 2;
}

int ktb_mlp_bf16(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                 const void* W2, const void* W3, void* logits, void* scratch, uintptr_t stream) {
  const MlpParams p{W1, nullptr, W2, nullptr, W3, nullptr, HeadKind::kGreedy, {logits}, true};
  return mlp_run("ktb_mlp_bf16", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, nullptr), scratch, stream);
}

int ktb_mlp_bf16_staged(int dev, const void* obs_peer, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                        const void* W2, const void* W3, void* logits, void* scratch, void* stage, uintptr_t stream) {
  KTB_REQUIRE(stage, KTB_ERR_ARG, "ktb_mlp_bf16_staged: null stage buffer");
  const MlpParams p{W1, nullptr, W2, nullptr, W3, nullptr, HeadKind::kGreedy, {logits}, true};
  return mlp_run("ktb_mlp_bf16_staged", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs_peer, stage), scratch,
                 stream);
}

int ktb_mlp_bf16_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_out,
                        const void* W1, const void* W2, const void* W3, void* logits, void* scratch, void* ctrl_local,
                        void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p{W1, nullptr, W2, nullptr, W3, nullptr, HeadKind::kGreedy, {logits}, true};
  return mlp_run("ktb_mlp_bf16_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                        const void* b1, const void* W2, const void* b2, const void* W3, const void* b3, void* logits,
                        int64_t* actions, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGreedy, {logits, actions}};
  return mlp_run("ktb_mlp_bf16_policy", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden,
                               int d_out, const void* W1, const void* b1, const void* W2, const void* b2,
                               const void* W3, const void* b3, void* logits, int64_t* actions, void* scratch,
                               void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                               unsigned long long seq, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGreedy, {logits, actions}};
  return mlp_run("ktb_mlp_bf16_policy_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                               const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                               const uint8_t* mask, void* logits, int64_t* actions, void* scratch, void* stage,
                               uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3, b3, HeadKind::kGreedy, {logits, actions}}.with_mask(mask);
  return mlp_run("ktb_mlp_bf16_policy_masked", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                      int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                      const void* b2, const void* W3, const void* b3, size_t mask_offset, void* logits,
                                      int64_t* actions, void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                      size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3, b3, HeadKind::kGreedy, {logits, actions}}.with_mask(nullptr);
  return mlp_run("ktb_mlp_bf16_policy_masked_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_sample(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                               const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                               uint64_t seed, uint64_t row_base, int64_t* actions, float* log_probs, void* scratch,
                               void* stage, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}};
  return mlp_run("ktb_mlp_bf16_policy_sample", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_sample_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                      int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                      const void* b2, const void* W3, const void* b3, uint64_t seed, uint64_t row_base,
                                      int64_t* actions, float* log_probs, void* scratch, void* ctrl_local,
                                      void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq,
                                      uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}};
  return mlp_run("ktb_mlp_bf16_policy_sample_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_sample_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                      const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                      const void* b3, const uint8_t* mask, uint64_t seed, uint64_t row_base,
                                      int64_t* actions, float* log_probs, void* scratch, void* stage,
                                      uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}}
                          .with_mask(mask);
  return mlp_run("ktb_mlp_bf16_policy_sample_masked", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_sample_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                             int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                             const void* b2, const void* W3, const void* b3, size_t mask_offset,
                                             uint64_t seed, uint64_t row_base, int64_t* actions, float* log_probs,
                                             void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                             size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3, b3, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}}
                          .with_mask(nullptr);
  return mlp_run("ktb_mlp_bf16_policy_sample_masked_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                 const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                                 const float* log_std, uint64_t seed, uint64_t row_base, float* actions,
                                 float* log_probs, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGaussian,
                    {nullptr, nullptr, log_probs, seed, row_base, log_std, actions}};
  return mlp_run("ktb_mlp_bf16_policy_gaussian", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_gaussian_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                        int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                        const void* b2, const void* W3, const void* b3, const float* log_std,
                                        uint64_t seed, uint64_t row_base, float* actions, float* log_probs,
                                        void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                        size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p{W1, b1, W2, b2, W3, b3, HeadKind::kGaussian,
                    {nullptr, nullptr, log_probs, seed, row_base, log_std, actions}};
  return mlp_run("ktb_mlp_bf16_policy_gaussian_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_sample_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                     const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v,
                                     const void* b3v, uint64_t seed, uint64_t row_base, int64_t* actions,
                                     float* log_probs, float* values, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3v, b3v, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}}
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_value", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_sample_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                            int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                            const void* b2, const void* W3v, const void* b3v, uint64_t seed,
                                            uint64_t row_base, int64_t* actions, float* log_probs, float* values,
                                            void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                            size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3v, b3v, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}}
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_sample_masked_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                            const void* W1, const void* b1, const void* W2, const void* b2,
                                            const void* W3v, const void* b3v, const uint8_t* mask, uint64_t seed,
                                            uint64_t row_base, int64_t* actions, float* log_probs, float* values,
                                            void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3v, b3v, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}}
                          .with_mask(mask)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_masked_value", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_sample_masked_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                   int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                   const void* W2, const void* b2, const void* W3v, const void* b3v,
                                                   size_t mask_offset, uint64_t seed, uint64_t row_base,
                                                   int64_t* actions, float* log_probs, float* values, void* scratch,
                                                   void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                   unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3v, b3v, HeadKind::kSample, {nullptr, actions, log_probs, seed, row_base}}
                          .with_mask(nullptr)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_masked_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v,
                                       const void* b3v, const float* log_std, uint64_t seed, uint64_t row_base,
                                       float* actions, float* log_probs, float* values, void* scratch, void* stage,
                                       uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3v, b3v, HeadKind::kGaussian,
                                {nullptr, nullptr, log_probs, seed, row_base, log_std, actions}}
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_value", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                              int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                              const void* b2, const void* W3v, const void* b3v, const float* log_std,
                                              uint64_t seed, uint64_t row_base, float* actions, float* log_probs,
                                              float* values, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                              int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams{W1, b1, W2, b2, W3v, b3v, HeadKind::kGaussian,
                                {nullptr, nullptr, log_probs, seed, row_base, log_std, actions}}
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_gaussian_state(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3s,
                                       const void* b3s, float log_std_min, float log_std_max, int squash,
                                       uint64_t seed, uint64_t row_base, float* actions, float* log_probs,
                                       void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::gaussian_state(W1, b1, W2, b2, W3s, b3s, log_std_min, log_std_max, squash,
                                                {nullptr, nullptr, log_probs, seed, row_base, nullptr, actions});
  return mlp_run("ktb_mlp_bf16_policy_gaussian_state", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_state_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                              int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                              const void* b2, const void* W3s, const void* b3s, float log_std_min,
                                              float log_std_max, int squash, uint64_t seed, uint64_t row_base,
                                              float* actions, float* log_probs, void* scratch, void* ctrl_local,
                                              void* ctrl_root_peer, int rank, size_t chunk_rows,
                                              unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::gaussian_state(W1, b1, W2, b2, W3s, b3s, log_std_min, log_std_max, squash,
                                                {nullptr, nullptr, log_probs, seed, row_base, nullptr, actions});
  return mlp_run("ktb_mlp_bf16_policy_gaussian_state_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_gaussian_state_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                             const void* W1, const void* b1, const void* W2, const void* b2,
                                             const void* W3sv, const void* b3sv, float log_std_min, float log_std_max,
                                             int squash, uint64_t seed, uint64_t row_base, float* actions,
                                             float* log_probs, float* values, void* scratch, void* stage,
                                             uintptr_t stream) {
  const MlpParams p = MlpParams::gaussian_state(W1, b1, W2, b2, W3sv, b3sv, log_std_min, log_std_max, squash,
                                                {nullptr, nullptr, log_probs, seed, row_base, nullptr, actions})
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_state_value", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_state_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                    int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                    const void* W2, const void* b2, const void* W3sv,
                                                    const void* b3sv, float log_std_min, float log_std_max, int squash,
                                                    uint64_t seed, uint64_t row_base, float* actions,
                                                    float* log_probs, float* values, void* scratch, void* ctrl_local,
                                                    void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                    unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::gaussian_state(W1, b1, W2, b2, W3sv, b3sv, log_std_min, log_std_max, squash,
                                                {nullptr, nullptr, log_probs, seed, row_base, nullptr, actions})
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_state_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_multidiscrete(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                      const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                      const void* b3, const int32_t* nvec, int n_groups, void* logits,
                                      int64_t* actions, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups, {logits, actions}, true);
  return mlp_run("ktb_mlp_bf16_policy_multidiscrete", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_multidiscrete_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                             int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                             const void* b2, const void* W3, const void* b3, const int32_t* nvec,
                                             int n_groups, void* logits, int64_t* actions, void* scratch,
                                             void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                             unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups, {logits, actions}, true);
  return mlp_run("ktb_mlp_bf16_policy_multidiscrete_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_multidiscrete_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                             const void* W1, const void* b1, const void* W2, const void* b2,
                                             const void* W3, const void* b3, const int32_t* nvec, int n_groups,
                                             const uint8_t* mask, void* logits, int64_t* actions, void* scratch,
                                             void* stage, uintptr_t stream) {
  const MlpParams p =
      MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups, {logits, actions}, true).with_mask(mask);
  return mlp_run("ktb_mlp_bf16_policy_multidiscrete_masked", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_multidiscrete_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                    int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                    const void* W2, const void* b2, const void* W3, const void* b3,
                                                    const int32_t* nvec, int n_groups, size_t mask_offset,
                                                    void* logits, int64_t* actions, void* scratch, void* ctrl_local,
                                                    void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                    unsigned long long seq, uintptr_t stream) {
  const MlpParams p =
      MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups, {logits, actions}, true).with_mask(nullptr);
  return mlp_run("ktb_mlp_bf16_policy_multidiscrete_masked_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                             const void* W1, const void* b1, const void* W2, const void* b2,
                                             const void* W3, const void* b3, const int32_t* nvec, int n_groups,
                                             uint64_t seed, uint64_t row_base, int64_t* actions, float* log_probs,
                                             void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                    int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                    const void* W2, const void* b2, const void* W3, const void* b3,
                                                    const int32_t* nvec, int n_groups, uint64_t seed,
                                                    uint64_t row_base, int64_t* actions, float* log_probs,
                                                    void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                                    size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden,
                                                    int d_out, const void* W1, const void* b1, const void* W2,
                                                    const void* b2, const void* W3, const void* b3,
                                                    const int32_t* nvec, int n_groups, const uint8_t* mask,
                                                    uint64_t seed, uint64_t row_base, int64_t* actions,
                                                    float* log_probs, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false)
                          .with_mask(mask);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete_masked", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete_masked_pushed(int dev, const void* stage_local, size_t stage_stride,
                                                           size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                                           const void* b1, const void* W2, const void* b2,
                                                           const void* W3, const void* b3, const int32_t* nvec,
                                                           int n_groups, size_t mask_offset, uint64_t seed,
                                                           uint64_t row_base, int64_t* actions, float* log_probs,
                                                           void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                                           int rank, size_t chunk_rows, unsigned long long seq,
                                                           uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3, b3, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false)
                          .with_mask(nullptr);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete_masked_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete_value(int dev, const void* obs, size_t M, int d_in, int d_hidden,
                                                   int d_out, const void* W1, const void* b1, const void* W2,
                                                   const void* b2, const void* W3v, const void* b3v,
                                                   const int32_t* nvec, int n_groups, uint64_t seed,
                                                   uint64_t row_base, int64_t* actions, float* log_probs,
                                                   float* values, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3v, b3v, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete_value", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete_value_pushed(int dev, const void* stage_local, size_t stage_stride,
                                                          size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                                          const void* b1, const void* W2, const void* b2,
                                                          const void* W3v, const void* b3v, const int32_t* nvec,
                                                          int n_groups, uint64_t seed, uint64_t row_base,
                                                          int64_t* actions, float* log_probs, float* values,
                                                          void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                                          int rank, size_t chunk_rows, unsigned long long seq,
                                                          uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3v, b3v, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete_masked_value(int dev, const void* obs, size_t M, int d_in, int d_hidden,
                                                          int d_out, const void* W1, const void* b1, const void* W2,
                                                          const void* b2, const void* W3v, const void* b3v,
                                                          const int32_t* nvec, int n_groups, const uint8_t* mask,
                                                          uint64_t seed, uint64_t row_base, int64_t* actions,
                                                          float* log_probs, float* values, void* scratch, void* stage,
                                                          uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3v, b3v, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false)
                          .with_mask(mask)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete_masked_value", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_sample_multidiscrete_masked_value_pushed(
    int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_out,
    const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v, const void* b3v,
    const int32_t* nvec, int n_groups, size_t mask_offset, uint64_t seed, uint64_t row_base, int64_t* actions,
    float* log_probs, float* values, void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
    size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::multidiscrete(W1, b1, W2, b2, W3v, b3v, nvec, n_groups,
                                               {nullptr, actions, log_probs, seed, row_base}, false)
                          .with_mask(nullptr)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_sample_multidiscrete_masked_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_epsilon_greedy(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                       const void* b3, const float* epsilon, uint64_t seed, uint64_t row_base,
                                       int64_t* actions, float* q, float* q_max, void* scratch, void* stage,
                                       uintptr_t stream) {
  const MlpParams p = MlpParams::epsilon_greedy(W1, b1, W2, b2, W3, b3, epsilon, seed, row_base, actions, q, q_max);
  return mlp_run("ktb_mlp_bf16_policy_epsilon_greedy", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_epsilon_greedy_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                              int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                              const void* b2, const void* W3, const void* b3, size_t epsilon_offset,
                                              uint64_t seed, uint64_t row_base, int64_t* actions, float* q,
                                              float* q_max, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                              int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::epsilon_greedy(W1, b1, W2, b2, W3, b3, nullptr, seed, row_base, actions, q, q_max);
  return mlp_run("ktb_mlp_bf16_policy_epsilon_greedy_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("epsilon", epsilon_offset, 4, 4),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_epsilon_greedy_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                              const void* W1, const void* b1, const void* W2, const void* b2,
                                              const void* W3, const void* b3, const uint8_t* mask,
                                              const float* epsilon, uint64_t seed, uint64_t row_base,
                                              int64_t* actions, float* q, float* q_max, void* scratch, void* stage,
                                              uintptr_t stream) {
  const MlpParams p =
      MlpParams::epsilon_greedy(W1, b1, W2, b2, W3, b3, epsilon, seed, row_base, actions, q, q_max).with_mask(mask);
  return mlp_run("ktb_mlp_bf16_policy_epsilon_greedy_masked", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_epsilon_greedy_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                     int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                     const void* W2, const void* b2, const void* W3, const void* b3,
                                                     size_t mask_offset, size_t epsilon_offset, uint64_t seed,
                                                     uint64_t row_base, int64_t* actions, float* q, float* q_max,
                                                     void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                                     size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p =
      MlpParams::epsilon_greedy(W1, b1, W2, b2, W3, b3, nullptr, seed, row_base, actions, q, q_max).with_mask(nullptr);
  return mlp_run("ktb_mlp_bf16_policy_epsilon_greedy_masked_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1)
                     .with_side("epsilon", epsilon_offset, 4, 4),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                 const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                                 const int32_t* nvec, int n_groups, const int64_t* taken, float* log_probs,
                                 float* entropy, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p =
      MlpParams::evaluate_categorical(W1, b1, W2, b2, W3, b3, nvec, n_groups, taken, log_probs, entropy);
  return mlp_run("ktb_mlp_bf16_policy_evaluate", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                        int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                        const void* b2, const void* W3, const void* b3, const int32_t* nvec,
                                        int n_groups, size_t taken_offset, float* log_probs, float* entropy,
                                        void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                        size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p =
      MlpParams::evaluate_categorical(W1, b1, W2, b2, W3, b3, nvec, n_groups, nullptr, log_probs, entropy);
  return mlp_run("ktb_mlp_bf16_policy_evaluate_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("taken", taken_offset, 8 * (size_t)std::max(n_groups, 1), 8),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v,
                                       const void* b3v, const int32_t* nvec, int n_groups, const int64_t* taken,
                                       float* log_probs, float* entropy, float* values, void* scratch, void* stage,
                                       uintptr_t stream) {
  const MlpParams p =
      MlpParams::evaluate_categorical(W1, b1, W2, b2, W3v, b3v, nvec, n_groups, taken, log_probs, entropy)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_evaluate_value", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                              int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                              const void* W2, const void* b2, const void* W3v, const void* b3v,
                                              const int32_t* nvec, int n_groups, size_t taken_offset, float* log_probs,
                                              float* entropy, float* values, void* scratch, void* ctrl_local,
                                              void* ctrl_root_peer, int rank, size_t chunk_rows,
                                              unsigned long long seq, uintptr_t stream) {
  const MlpParams p =
      MlpParams::evaluate_categorical(W1, b1, W2, b2, W3v, b3v, nvec, n_groups, nullptr, log_probs, entropy)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_evaluate_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("taken", taken_offset, 8 * (size_t)std::max(n_groups, 1), 8),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                        const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                        const void* b3, const int32_t* nvec, int n_groups, const uint8_t* mask,
                                        const int64_t* taken, float* log_probs, float* entropy, void* scratch,
                                        void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::evaluate_categorical(W1, b1, W2, b2, W3, b3, nvec, n_groups, taken, log_probs, entropy)
                          .with_mask(mask);
  return mlp_run("ktb_mlp_bf16_policy_evaluate_masked", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                               int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                               const void* W2, const void* b2, const void* W3, const void* b3,
                                               const int32_t* nvec, int n_groups, size_t mask_offset,
                                               size_t taken_offset, float* log_probs, float* entropy, void* scratch,
                                               void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                               unsigned long long seq, uintptr_t stream) {
  const MlpParams p =
      MlpParams::evaluate_categorical(W1, b1, W2, b2, W3, b3, nvec, n_groups, nullptr, log_probs, entropy)
                          .with_mask(nullptr);
  return mlp_run("ktb_mlp_bf16_policy_evaluate_masked_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1)
                     .with_side("taken", taken_offset, 8 * (size_t)std::max(n_groups, 1), 8),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate_masked_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                              const void* W1, const void* b1, const void* W2, const void* b2,
                                              const void* W3v, const void* b3v, const int32_t* nvec, int n_groups,
                                              const uint8_t* mask, const int64_t* taken, float* log_probs,
                                              float* entropy, float* values, void* scratch, void* stage,
                                              uintptr_t stream) {
  const MlpParams p =
      MlpParams::evaluate_categorical(W1, b1, W2, b2, W3v, b3v, nvec, n_groups, taken, log_probs, entropy)
                          .with_mask(mask)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_evaluate_masked_value", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_evaluate_masked_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                     int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                     const void* W2, const void* b2, const void* W3v, const void* b3v,
                                                     const int32_t* nvec, int n_groups, size_t mask_offset,
                                                     size_t taken_offset, float* log_probs, float* entropy,
                                                     float* values, void* scratch, void* ctrl_local,
                                                     void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                     unsigned long long seq, uintptr_t stream) {
  const MlpParams p =
      MlpParams::evaluate_categorical(W1, b1, W2, b2, W3v, b3v, nvec, n_groups, nullptr, log_probs, entropy)
                          .with_mask(nullptr)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_evaluate_masked_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("mask", mask_offset, d_out, 1)
                     .with_side("taken", taken_offset, 8 * (size_t)std::max(n_groups, 1), 8),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_evaluate(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                          const void* W1, const void* b1, const void* W2, const void* b2,
                                          const void* W3, const void* b3, const float* log_std, const float* taken,
                                          float* log_probs, float* entropy, void* scratch, void* stage,
                                          uintptr_t stream) {
  const MlpParams p = MlpParams::evaluate_gaussian(W1, b1, W2, b2, W3, b3, log_std, taken, log_probs, entropy);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_evaluate", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_evaluate_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                 int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                 const void* W2, const void* b2, const void* W3, const void* b3,
                                                 const float* log_std, size_t taken_offset, float* log_probs,
                                                 float* entropy, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                                 int rank, size_t chunk_rows, unsigned long long seq,
                                                 uintptr_t stream) {
  const MlpParams p = MlpParams::evaluate_gaussian(W1, b1, W2, b2, W3, b3, log_std, nullptr, log_probs, entropy);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_evaluate_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("taken", taken_offset, 4 * (size_t)d_out, 4),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_evaluate_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                                const void* W1, const void* b1, const void* W2, const void* b2,
                                                const void* W3v, const void* b3v, const float* log_std,
                                                const float* taken, float* log_probs, float* entropy, float* values,
                                                void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::evaluate_gaussian(W1, b1, W2, b2, W3v, b3v, log_std, taken, log_probs, entropy)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_evaluate_value", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_policy_gaussian_evaluate_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                       int d_in, int d_hidden, int d_out, const void* W1,
                                                       const void* b1, const void* W2, const void* b2, const void* W3v,
                                                       const void* b3v, const float* log_std, size_t taken_offset,
                                                       float* log_probs, float* entropy, float* values, void* scratch,
                                                       void* ctrl_local, void* ctrl_root_peer, int rank,
                                                       size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::evaluate_gaussian(W1, b1, W2, b2, W3v, b3v, log_std, nullptr, log_probs, entropy)
                          .with_values(values);
  return mlp_run("ktb_mlp_bf16_policy_gaussian_evaluate_value_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("taken", taken_offset, 4 * (size_t)d_out, 4),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_deterministic(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                      const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                      const void* b3, float noise, float noise_clip, int squash, uint64_t seed,
                                      uint64_t row_base, float* actions, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p =
      MlpParams::deterministic(W1, b1, W2, b2, W3, b3, noise, noise_clip, squash, seed, row_base, actions);
  return mlp_run("ktb_mlp_bf16_policy_deterministic", dev, M, d_in, d_hidden, d_out, p, MlpFeed::pull(obs, stage),
                 scratch, stream);
}

int ktb_mlp_bf16_policy_deterministic_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                             int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                             const void* b2, const void* W3, const void* b3, float noise,
                                             float noise_clip, int squash, uint64_t seed, uint64_t row_base,
                                             float* actions, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                             int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams p =
      MlpParams::deterministic(W1, b1, W2, b2, W3, b3, noise, noise_clip, squash, seed, row_base, actions);
  return mlp_run("ktb_mlp_bf16_policy_deterministic_pushed", dev, M, d_in, d_hidden, d_out, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq), scratch,
                 stream);
}

int ktb_mlp_bf16_critic(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act, const void* W1p,
                        const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                        const float* act, float* q, void* scratch, void* stage, uintptr_t stream) {
  const MlpParams p = MlpParams::critic_head(W1p, b1, W2, b2, W3, b3, d_act, act, q);
  return mlp_run("ktb_mlp_bf16_critic", dev, M, d_in, d_hidden, 1, p, MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_critic_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden,
                               int d_act, const void* W1p, const void* b1, const void* W2, const void* b2,
                               const void* W3, const void* b3, size_t act_offset, float* q, void* scratch,
                               void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                               unsigned long long seq, uintptr_t stream) {
  const MlpParams p = MlpParams::critic_head(W1p, b1, W2, b2, W3, b3, d_act, nullptr, q);
  return mlp_run("ktb_mlp_bf16_critic_pushed", dev, M, d_in, d_hidden, 1, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("act", act_offset, 4 * (size_t)d_act, 4),
                 scratch, stream);
}

int ktb_mlp_bf16_critic_twin(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act, const void* W1p,
                             const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                             const void* W1p_2, const void* b1_2, const void* W2_2, const void* b2_2,
                             const void* W3_2, const void* b3_2, const float* act, float* q1, float* q2, float* q_min,
                             void* scratch, void* stage, uintptr_t stream) {
  MlpParams second = MlpParams::critic_head(W1p_2, b1_2, W2_2, b2_2, W3_2, b3_2, d_act, act, q2);
  second.hq.q_other = q1;
  second.hq.q_min = q_min;
  MlpParams p = MlpParams::critic_head(W1p, b1, W2, b2, W3, b3, d_act, act, q1);
  p.twin = &second;
  return mlp_run("ktb_mlp_bf16_critic_twin", dev, M, d_in, d_hidden, 1, p, MlpFeed::pull(obs, stage), scratch,
                 stream);
}

int ktb_mlp_bf16_critic_twin_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                    int d_hidden, int d_act, const void* W1p, const void* b1, const void* W2,
                                    const void* b2, const void* W3, const void* b3, const void* W1p_2,
                                    const void* b1_2, const void* W2_2, const void* b2_2, const void* W3_2,
                                    const void* b3_2, size_t act_offset, float* q1, float* q2, float* q_min,
                                    void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                    unsigned long long seq, uintptr_t stream) {
  MlpParams second = MlpParams::critic_head(W1p_2, b1_2, W2_2, b2_2, W3_2, b3_2, d_act, nullptr, q2);
  second.hq.q_other = q1;
  second.hq.q_min = q_min;
  MlpParams p = MlpParams::critic_head(W1p, b1, W2, b2, W3, b3, d_act, nullptr, q1);
  p.twin = &second;
  return mlp_run("ktb_mlp_bf16_critic_twin_pushed", dev, M, d_in, d_hidden, 1, p,
                 MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                     .with_side("act", act_offset, 4 * (size_t)d_act, 4),
                 scratch, stream);
}

size_t ktb_mlp_td_target_scratch_bytes(size_t M, int d_hidden_actor, int d_hidden, int d_act) {
  const size_t rows = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  return ktb_mlp_critic_scratch_bytes(M, std::max(d_hidden_actor, d_hidden)) + rows * (4 * (size_t)d_act + 8);
}

size_t ktb_mlp_dqn_target_scratch_bytes(size_t M, int d_hidden) {
  const size_t rows = std::min<size_t>(M, (size_t)g_mlp_chunk_rows);
  return ktb_mlp_scratch_bytes(M, d_hidden) + rows * 8;
}

}  // extern "C"

namespace ktb {

// The critics of a TD target (the first and, unless the six pointers of the second are all null, a twin's second)
// over the actions of `actor`, the last one's HeadQ holding the target's inputs and output; mlp_run points their
// scratch pointers into the chunk scratch.  A partly given second critic is a twin with a null weight, which mlp_run
// refuses.
static int td_target_run(const char* fn, int dev, size_t M, int d_in, int d_hidden, int d_act, const void* const (&c)[12],
                         int d_hidden_actor, const MlpParams& actor, const float* reward, const float* done,
                         float gamma, float alpha, float* y, const MlpFeed& f, void* scratch, uintptr_t stream) {
  MlpParams second = MlpParams::critic_head(c[6], c[7], c[8], c[9], c[10], c[11], d_act, nullptr, nullptr);
  MlpParams p = MlpParams::critic_head(c[0], c[1], c[2], c[3], c[4], c[5], d_act, nullptr, nullptr);
  if (std::any_of(c + 6, c + 12, [](const void* x) { return x != nullptr; })) p.twin = &second;
  HeadQ& t = (p.twin ? second : p).hq;
  t.reward = reward;
  t.done = done;
  t.y = y;
  t.gamma = gamma;
  t.alpha = alpha;
  p.target = second.target = true;
  p.actor = &actor;
  p.actor_hidden = d_hidden_actor;
  return mlp_run(fn, dev, M, d_in, d_hidden, 1, p, f, scratch, stream);
}

// A DQN target: the target network (w[0..5]) in the kSample instantiations, whose hq computes y, and unless the six
// pointers w[6..11] are all null Double DQN's online network, a greedy head; `masked` marks the _masked entries (mask
// null in the pushed forms).  A partly given online network has a null weight, which mlp_run refuses.
static int dqn_target_run(const char* fn, int dev, size_t M, int d_in, int d_hidden, int d_out,
                          const void* const (&w)[12], bool masked, const uint8_t* mask, const float* reward,
                          const float* done, float gamma, float* y, const MlpFeed& f, void* scratch, uintptr_t stream) {
  const MlpParams online{w[6], w[7], w[8], w[9], w[10], w[11], HeadKind::kGreedy};
  MlpParams p{w[0], w[1], w[2], w[3], w[4], w[5], HeadKind::kSample};
  if (masked) p = p.with_mask(mask);
  if (std::any_of(w + 6, w + 12, [](const void* x) { return x != nullptr; })) p.online = &online;
  p.dqn = p.target = true;
  p.hq.reward = reward;
  p.hq.done = done;
  p.hq.gamma = gamma;
  p.hq.y = y;
  return mlp_run(fn, dev, M, d_in, d_hidden, d_out, p, f, scratch, stream);
}

}  // namespace ktb

extern "C" {

int ktb_mlp_bf16_td_target_deterministic(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act,
                                         const void* W1p, const void* b1, const void* W2, const void* b2,
                                         const void* W3, const void* b3, const void* W1p_2, const void* b1_2,
                                         const void* W2_2, const void* b2_2, const void* W3_2, const void* b3_2,
                                         int d_hidden_actor, const void* aW1, const void* ab1, const void* aW2,
                                         const void* ab2, const void* aW3, const void* ab3, float noise,
                                         float noise_clip, int squash, uint64_t seed, uint64_t row_base,
                                         const float* reward, const float* done, float gamma, float* y, void* scratch,
                                         void* stage, uintptr_t stream) {
  const MlpParams a =
      MlpParams::deterministic(aW1, ab1, aW2, ab2, aW3, ab3, noise, noise_clip, squash, seed, row_base, nullptr);
  return td_target_run("ktb_mlp_bf16_td_target_deterministic", dev, M, d_in, d_hidden, d_act,
                       {W1p, b1, W2, b2, W3, b3, W1p_2, b1_2, W2_2, b2_2, W3_2, b3_2}, d_hidden_actor, a, reward, done,
                       gamma, 0.f, y, MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_td_target_deterministic_pushed(
    int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_act,
    const void* W1p, const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
    const void* W1p_2, const void* b1_2, const void* W2_2, const void* b2_2, const void* W3_2, const void* b3_2,
    int d_hidden_actor, const void* aW1, const void* ab1, const void* aW2, const void* ab2, const void* aW3,
    const void* ab3, float noise, float noise_clip, int squash, uint64_t seed, uint64_t row_base,
    size_t reward_offset, size_t done_offset, float gamma, float* y, void* scratch, void* ctrl_local,
    void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams a =
      MlpParams::deterministic(aW1, ab1, aW2, ab2, aW3, ab3, noise, noise_clip, squash, seed, row_base, nullptr);
  return td_target_run("ktb_mlp_bf16_td_target_deterministic_pushed", dev, M, d_in, d_hidden, d_act,
                       {W1p, b1, W2, b2, W3, b3, W1p_2, b1_2, W2_2, b2_2, W3_2, b3_2}, d_hidden_actor, a, nullptr,
                       nullptr, gamma, 0.f, y,
                       MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                           .with_side("reward", reward_offset, 4, 4).with_side("done", done_offset, 4, 4),
                       scratch, stream);
}

int ktb_mlp_bf16_td_target_gaussian(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act,
                                    const void* W1p, const void* b1, const void* W2, const void* b2, const void* W3,
                                    const void* b3, const void* W1p_2, const void* b1_2, const void* W2_2,
                                    const void* b2_2, const void* W3_2, const void* b3_2, int d_hidden_actor,
                                    const void* aW1, const void* ab1, const void* aW2, const void* ab2,
                                    const void* aW3s, const void* ab3s, float log_std_min, float log_std_max,
                                    int squash, uint64_t seed, uint64_t row_base, const float* reward,
                                    const float* done, float gamma, float alpha, float* y, void* scratch, void* stage,
                                    uintptr_t stream) {
  const MlpParams a = MlpParams::gaussian_state(aW1, ab1, aW2, ab2, aW3s, ab3s, log_std_min, log_std_max, squash,
                                                {nullptr, nullptr, nullptr, seed, row_base});
  return td_target_run("ktb_mlp_bf16_td_target_gaussian", dev, M, d_in, d_hidden, d_act,
                       {W1p, b1, W2, b2, W3, b3, W1p_2, b1_2, W2_2, b2_2, W3_2, b3_2}, d_hidden_actor, a, reward, done,
                       gamma, alpha, y, MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_td_target_gaussian_pushed(
    int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_act,
    const void* W1p, const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
    const void* W1p_2, const void* b1_2, const void* W2_2, const void* b2_2, const void* W3_2, const void* b3_2,
    int d_hidden_actor, const void* aW1, const void* ab1, const void* aW2, const void* ab2, const void* aW3s,
    const void* ab3s, float log_std_min, float log_std_max, int squash, uint64_t seed, uint64_t row_base,
    size_t reward_offset, size_t done_offset, float gamma, float alpha, float* y, void* scratch, void* ctrl_local,
    void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  const MlpParams a = MlpParams::gaussian_state(aW1, ab1, aW2, ab2, aW3s, ab3s, log_std_min, log_std_max, squash,
                                                {nullptr, nullptr, nullptr, seed, row_base});
  return td_target_run("ktb_mlp_bf16_td_target_gaussian_pushed", dev, M, d_in, d_hidden, d_act,
                       {W1p, b1, W2, b2, W3, b3, W1p_2, b1_2, W2_2, b2_2, W3_2, b3_2}, d_hidden_actor, a, nullptr,
                       nullptr, gamma, alpha, y,
                       MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                           .with_side("reward", reward_offset, 4, 4).with_side("done", done_offset, 4, 4),
                       scratch, stream);
}

int ktb_mlp_bf16_dqn_target(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                            const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                            const void* oW1, const void* ob1, const void* oW2, const void* ob2, const void* oW3,
                            const void* ob3, const float* reward, const float* done, float gamma, float* y,
                            void* scratch, void* stage, uintptr_t stream) {
  return dqn_target_run("ktb_mlp_bf16_dqn_target", dev, M, d_in, d_hidden, d_out,
                        {W1, b1, W2, b2, W3, b3, oW1, ob1, oW2, ob2, oW3, ob3}, false, nullptr, reward, done, gamma, y,
                        MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_dqn_target_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                   int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                   const void* b2, const void* W3, const void* b3, const void* oW1, const void* ob1,
                                   const void* oW2, const void* ob2, const void* oW3, const void* ob3,
                                   size_t rd_offset, float gamma, float* y, void* scratch, void* ctrl_local,
                                   void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq,
                                   uintptr_t stream) {
  return dqn_target_run("ktb_mlp_bf16_dqn_target_pushed", dev, M, d_in, d_hidden, d_out,
                        {W1, b1, W2, b2, W3, b3, oW1, ob1, oW2, ob2, oW3, ob3}, false, nullptr, nullptr, nullptr, gamma,
                        y,
                        MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                            .with_side("rd", rd_offset, 8, 8),
                        scratch, stream);
}

int ktb_mlp_bf16_dqn_target_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                   const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                   const void* b3, const void* oW1, const void* ob1, const void* oW2, const void* ob2,
                                   const void* oW3, const void* ob3, const uint8_t* mask, const float* reward,
                                   const float* done, float gamma, float* y, void* scratch, void* stage,
                                   uintptr_t stream) {
  return dqn_target_run("ktb_mlp_bf16_dqn_target_masked", dev, M, d_in, d_hidden, d_out,
                        {W1, b1, W2, b2, W3, b3, oW1, ob1, oW2, ob2, oW3, ob3}, true, mask, reward, done, gamma, y,
                        MlpFeed::pull(obs, stage), scratch, stream);
}

int ktb_mlp_bf16_dqn_target_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                          int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                          const void* b2, const void* W3, const void* b3, const void* oW1,
                                          const void* ob1, const void* oW2, const void* ob2, const void* oW3,
                                          const void* ob3, size_t mask_offset, size_t rd_offset, float gamma, float* y,
                                          void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                          size_t chunk_rows, unsigned long long seq, uintptr_t stream) {
  return dqn_target_run("ktb_mlp_bf16_dqn_target_masked_pushed", dev, M, d_in, d_hidden, d_out,
                        {W1, b1, W2, b2, W3, b3, oW1, ob1, oW2, ob2, oW3, ob3}, true, nullptr, nullptr, nullptr, gamma,
                        y,
                        MlpFeed::push(stage_local, stage_stride, ctrl_local, ctrl_root_peer, rank, chunk_rows, seq)
                            .with_side("mask", mask_offset, d_out, 1)
                            .with_side("rd", rd_offset, 8, 8),
                        scratch, stream);
}

}  // extern "C"
