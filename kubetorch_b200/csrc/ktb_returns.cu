// ktb_returns.cu — the learner targets of env-major [N, T] rollouts, the reverse linear recurrences of include/ktb200.h
// evaluated exactly as written there:
//   ktb_gae_f32     generalized advantage estimation: PPO's advantages and λ-returns;
//   ktb_vtrace_f32  V-trace (IMPALA): off-policy value targets and policy-gradient advantages;
//   ktb_retrace_f32 Retrace(λ) (ACER, Reactor, MPO, Q(λ)): off-policy Q-value targets and their TD errors;
// and the n-step bootstrapped returns that are no recurrence along the row (nstep_kernel, after the first three):
//   ktb_nstep_f32   Ape-X's, R2D2's and A3C's n-step targets and their TD errors.
//
// HBM-bound: (4·inputs + 8)·N·T + 4·N bytes, a handful of flops per element.  The recurrence runs along a row, but the
// rows are stored env-major, so one thread per row would read with a stride of T elements.  Instead each warp owns 32
// rows and walks T backwards in 32-step tiles:
//   loads  for each of its rows the 32 lanes copy 32 consecutive steps of every input into shared tiles (cp.async, 4
//          bytes per lane: any T and any 4-byte alignment take the same path, and each row's 32 words are one
//          coalesced access), rows padded to 33 words so that the scan's column reads hit 32 banks;
//   scan   lane i runs row i's recurrence over the tile, right to left, with __fadd_rn / __fmul_rn / __fsub_rn so that
//          nothing is contracted into an FMA, and writes the two outputs over the tile's first two input planes;
//   stores the lanes write the tile's rows of both outputs back as consecutive steps.
// kStages tiles are in flight per warp: the loads of the next kStages - 1 (earlier) tiles are issued before the current
// one is scanned.  A tile shorter than 32 steps (T % 32 at the end of the row, or T < 32) is copied by flat index over
// its rows, so that small T still moves whole segments.  The tile walk is scan_rows(); each op is a per-step functor.
#include "ktb_common.cuh"

#include <atomic>
#include <cmath>

namespace ktb {

constexpr int kPad = 33;
constexpr int kGaeStages = 3;      // 3 x 12.4 KiB of shared tiles per warp (3 planes)
// 2 x 16.5 KiB per warp (4 planes), 6 blocks per SM, in dynamic shared memory.  Three stages (49.5 KiB, past the static
// limit) measured 0.4-2.5 % slower at every shape of tools/bench_vtrace.py: the per-step exp, not the loads, bounds long
// rows.  The same two stages as a static array compile to 114 registers instead of 80 and measured 1.8-4.1 % slower
// (DESIGN.md §4b).
constexpr int kVtraceStages = 2;
constexpr int kVtraceSmem = kVtraceStages * 4 * 32 * kPad * 4;   // 33 792 B: under 48 KiB, so no opt-in attribute
// 2 x 24.8 KiB per warp (6 planes), 4 blocks per SM: past 48 KiB, so the launch opts in to the larger dynamic size.
// Five planes under 48 KiB (42 240 B, 5 blocks per SM), td formed at store time from a coalesced read of baseline,
// measured 3.5 % and 8.8 % slower at (16384, 128) and (4096, 256) and at most 3 % faster at the latency-bound shapes of
// tools/bench_retrace.py; the same with the tile's baseline read into registers before the scan was 6-21 % slower at
// every shape (DESIGN.md §4b).
constexpr int kRetraceStages = 2;
constexpr int kRetraceSmem = kRetraceStages * 6 * 32 * kPad * 4;   // 50 688 B

template <int P>
using Tile = float[P][32][kPad];   // [input plane][row][step]

__device__ __forceinline__ void cp_async4(float* smem, const float* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// f(j, c) for every (row j < nr, step c < len) of a tile, one element per lane and call: row by row when the tile is
// full, by flat index over the rows otherwise.
template <class F>
__device__ __forceinline__ void for_tile(int nr, int len, int lane, F&& f) {
  if (len == 32) {
    for (int j = 0; j < nr; ++j) f(j, lane);
  } else {
    for (int e = lane; e < nr * len; e += 32) {
      const int j = e / len;
      f(j, e - j * len);
    }
  }
}

// The tile walk of one warp over its 32 rows: P input planes in[] staged through tile[kStages], step.start(boot[row])
// once per lane, then step(s, lane, c) for c = len - 1 … 0 of every tile, right to left; step leaves its two outputs
// in planes 0 and 1, which go to out0 and out1.
template <int P, int kStages, class Step>
__device__ __forceinline__ void scan_rows(Tile<P>* tile, const float* const (&in)[P], const float* boot, size_t N,
                                          size_t T, float* out0, float* out1, Step& step) {
  const int lane = threadIdx.x;
  const size_t row0 = (size_t)blockIdx.x * 32;
  const int nr = (int)(N - row0 < 32 ? N - row0 : 32);
  const size_t n_tiles = (T + 31) / 32;
  const size_t base = row0 * T;

  // tile k covers steps [t0, t0 + len) with k = 0 the last 32-aligned tile of the row
  auto t0_of = [&](size_t k) { return (n_tiles - 1 - k) * 32; };
  auto len_of = [&](size_t t0) { return (int)(T - t0 < 32 ? T - t0 : 32); };
  auto issue = [&](size_t k) {
    if (k < n_tiles) {
      const size_t t0 = t0_of(k);
      Tile<P>& s = tile[k % kStages];
      for_tile(nr, len_of(t0), lane, [&](int j, int c) {
        const size_t g = base + (size_t)j * T + t0 + c;
#pragma unroll
        for (int p = 0; p < P; ++p) cp_async4(&s[p][j][c], in[p] + g);
      });
    }
    cp_async_commit();   // one group per tile, empty past the first step: wait_group counts stay uniform
  };

  for (int k = 0; k < kStages - 1; ++k) issue(k);
  step.start(lane < nr ? boot[row0 + lane] : 0.0f);
  for (size_t k = 0; k < n_tiles; ++k) {
    issue(k + kStages - 1);
    cp_async_wait<kStages - 1>();   // this lane's copies of tile k have landed
    __syncwarp();                   // ... and every other lane's
    Tile<P>& s = tile[k % kStages];
    const size_t t0 = t0_of(k);
    const int len = len_of(t0);
    if (lane < nr) {
      for (int c = len - 1; c >= 0; --c) step(s, lane, c);
    }
    __syncwarp();
    for_tile(nr, len, lane, [&](int j, int c) {
      const size_t g = base + (size_t)j * T + t0 + c;
      out0[g] = s[0][j][c];
      out1[g] = s[1][j][c];
    });
    __syncwarp();   // the stage is reloaded by the next iteration's issue()
  }
}

// GAE over planes [rewards → adv, values → ret, dones].
struct GaeStep {
  float gamma, gamma_lam, acc, nv;
  __device__ __forceinline__ void start(float last_value) {
    acc = 0.0f;
    nv = last_value;
  }
  __device__ __forceinline__ void operator()(Tile<3>& s, int j, int c) {
    const float v = s[1][j][c];
    const float nt = __fsub_rn(1.0f, s[2][j][c]);
    const float delta = __fsub_rn(__fadd_rn(s[0][j][c], __fmul_rn(__fmul_rn(gamma, nv), nt)), v);
    acc = __fadd_rn(delta, __fmul_rn(__fmul_rn(gamma_lam, nt), acc));
    s[0][j][c] = acc;
    s[1][j][c] = __fadd_rn(acc, v);
    nv = v;
  }
};

// V-trace over planes [log_rhos → vs, rewards → pg_adv, values, dones].  The clips are compares, so that a NaN ρ stays
// NaN as under torch.clamp (fminf would return the threshold); a threshold of +inf never clips.
struct VtraceStep {
  float gamma, lam, rho_bar, c_bar, pg_rho_bar, acc, nv, nvs;
  __device__ __forceinline__ void start(float bootstrap) {
    acc = 0.0f;
    nv = nvs = bootstrap;
  }
  __device__ __forceinline__ void operator()(Tile<4>& s, int j, int c) {
    const float rho = expf(s[0][j][c]);
    const float r = s[1][j][c], v = s[2][j][c];
    const float disc = __fmul_rn(gamma, __fsub_rn(1.0f, s[3][j][c]));
    const float cr = rho > rho_bar ? rho_bar : rho;
    const float cc = __fmul_rn(lam, rho > c_bar ? c_bar : rho);
    const float pr = rho > pg_rho_bar ? pg_rho_bar : rho;
    const float delta = __fmul_rn(cr, __fsub_rn(__fadd_rn(r, __fmul_rn(disc, nv)), v));
    acc = __fadd_rn(delta, __fmul_rn(__fmul_rn(disc, cc), acc));
    const float vs = __fadd_rn(acc, v);
    s[0][j][c] = vs;
    s[1][j][c] = __fmul_rn(pr, __fsub_rn(__fadd_rn(r, __fmul_rn(disc, nvs)), v));
    nv = v;
    nvs = vs;
  }
};

// Retrace(λ) over planes [log_rhos → ret, rewards → td, q, values, dones, baseline].  The step carries the next step's
// value, Q and trace (nv, nq, nc); starting from nq = nc = −0 makes the general step reproduce the first one, r + disc ·
// bootstrap, bit for bit (−0 included).  The clip is a compare, so that a NaN ρ stays NaN as under torch.clamp.
struct RetraceStep {
  float gamma, lam, acc, nv, nq, nc;
  __device__ __forceinline__ void start(float bootstrap) {
    acc = 0.0f;
    nv = bootstrap;
    nq = nc = -0.0f;
  }
  __device__ __forceinline__ void operator()(Tile<6>& s, int j, int c) {
    const float rho = expf(s[0][j][c]);
    const float disc = __fmul_rn(gamma, __fsub_rn(1.0f, s[4][j][c]));
    acc = __fadd_rn(s[1][j][c], __fmul_rn(disc, __fadd_rn(__fsub_rn(nv, __fmul_rn(nc, nq)), __fmul_rn(nc, acc))));
    s[0][j][c] = acc;
    s[1][j][c] = __fsub_rn(acc, s[5][j][c]);
    nc = __fmul_rn(lam, rho > 1.0f ? 1.0f : rho);
    nv = s[3][j][c];
    nq = s[2][j][c];
  }
};

// One warp per block and per 32 rows.
__global__ void __launch_bounds__(32)
    gae_kernel(const float* __restrict__ rewards, const float* __restrict__ values, const float* __restrict__ dones,
               const float* __restrict__ last_values, size_t N, size_t T, float gamma, float gamma_lam,
               float* __restrict__ adv, float* __restrict__ ret) {
  __shared__ Tile<3> tile[kGaeStages];
  const float* const in[3] = {rewards, values, dones};
  GaeStep step{gamma, gamma_lam};
  scan_rows<3, kGaeStages>(tile, in, last_values, N, T, adv, ret, step);
}

__global__ void __launch_bounds__(32)
    vtrace_kernel(const float* __restrict__ log_rhos, const float* __restrict__ rewards,
                  const float* __restrict__ values, const float* __restrict__ dones,
                  const float* __restrict__ bootstrap, size_t N, size_t T, float gamma, float lam, float rho_bar,
                  float c_bar, float pg_rho_bar, float* __restrict__ vs, float* __restrict__ pg_adv) {
  extern __shared__ __align__(16) float smem[];
  const float* const in[4] = {log_rhos, rewards, values, dones};
  VtraceStep step{gamma, lam, rho_bar, c_bar, pg_rho_bar};
  scan_rows<4, kVtraceStages>(reinterpret_cast<Tile<4>*>(smem), in, bootstrap, N, T, vs, pg_adv, step);
}

__global__ void __launch_bounds__(32)
    retrace_kernel(const float* __restrict__ log_rhos, const float* __restrict__ rewards, const float* __restrict__ q,
                   const float* __restrict__ values, const float* __restrict__ dones,
                   const float* __restrict__ baseline, const float* __restrict__ bootstrap, size_t N, size_t T,
                   float gamma, float lam, float* __restrict__ ret, float* __restrict__ td) {
  extern __shared__ __align__(16) float smem[];
  const float* const in[6] = {log_rhos, rewards, q, values, dones, baseline};
  RetraceStep step{gamma, lam};
  scan_rows<6, kRetraceStages>(reinterpret_cast<Tile<6>*>(smem), in, bootstrap, N, T, ret, td, step);
}

// n-step bootstrapped returns.  Unlike the recurrences above, output (i, t) depends only on the window of steps
// [t, t + n] of its row, so the grid splits T as well as N: block (x, y) is one warp over rows [32x, 32x + 32) and the
// span of kNstepSpan consecutive 32-step tiles starting at tile y·span.  The warp walks its span forwards with a ring of
// two tiles per row in shared memory, the current one and the next (the windows' halo), so a tile copied as the halo is
// the next iteration's current tile and is read from global memory once; only the span's last halo is cut to the n
// steps the windows reach.  Steps past T hold the header's padding (reward 0, discount 1, value V(s_T)), so every
// window runs its n operations with no branch.  Lane c computes step t0 + c of kNstepRows rows at a time: its reads of
// ring position (c + k) & 63 are consecutive across the lanes (no bank conflicts), and the rows' chains interleave.
// One tile per warp and eight rows at a time measured fastest at three of the four shapes of tools/bench_nstep.py (one
// tile and four rows: 1-17 % slower; two tiles: up to 86 % slower, 2-8 % faster at (16384, 128); four: slower at
// every shape): the warp waits for its copies once per tile, so more warps beat a longer span (DESIGN.md §4b).  The
// span is larger only where T has more than 65535 tiles, the grid's y limit.
constexpr int kNstepSpan = 1;
constexpr int kNstepRows = 8;

__global__ void __launch_bounds__(32)
    nstep_kernel(const float* __restrict__ rewards, const float* __restrict__ values, const float* __restrict__ dones,
                 const float* __restrict__ baseline, const float* __restrict__ last_values, size_t N, size_t T, int n,
                 float gamma, size_t span, float* __restrict__ ret, float* __restrict__ td) {
  __shared__ __align__(16) float2 rd[32][64];   // [row][ring position]: (reward, gamma·(1 − done)), 16 KiB
  __shared__ float vv[32][64];                  // [row][ring position]: value, 8 KiB
  const int lane = threadIdx.x;
  const size_t row0 = (size_t)blockIdx.x * 32;
  const int nr = (int)(N - row0 < 32 ? N - row0 : 32);
  const size_t n_tiles = (T + 31) / 32;
  const size_t k0 = (size_t)blockIdx.y * span;
  const size_t k1 = k0 + span < n_tiles ? k0 + span : n_tiles;
  const size_t base = row0 * T;
  const float lv = lane < nr ? last_values[row0 + lane] : 0.0f;   // V(s_T) of row `lane`

  auto len_of = [&](size_t k) { return k < n_tiles ? (int)(T - k * 32 < 32 ? T - k * 32 : 32) : 0; };
  // the steps of tile k to copy: all of them inside the span, the n that the last windows reach past it
  auto count = [&](size_t k) { return k < k1 ? len_of(k) : min(len_of(k), n); };
  auto issue = [&](size_t k, int cnt) {
    const int p0 = (int)(k & 1) * 32;
    for_tile(nr, cnt, lane, [&](int j, int c) {
      const size_t g = base + (size_t)j * T + k * 32 + c;
      cp_async4(&rd[j][p0 + c].x, rewards + g);
      cp_async4(&rd[j][p0 + c].y, dones + g);
      cp_async4(&vv[j][p0 + c], values + g);
    });
  };
  // once tile k's copies have landed: the discount of each copied step, and the padding at every other position
  auto convert = [&](size_t k, int cnt) {
    const int p = (int)(k & 1) * 32 + lane;
    for (int j = 0; j < nr; ++j) {
      const float lvj = __shfl_sync(0xffffffffu, lv, j);
      if (lane < cnt) {
        rd[j][p].y = __fmul_rn(gamma, __fsub_rn(1.0f, rd[j][p].y));
      } else {
        rd[j][p] = make_float2(0.0f, 1.0f);
        vv[j][p] = lvj;
      }
    }
  };

  issue(k0, len_of(k0));
  for (size_t k = k0; k < k1; ++k) {
    issue(k + 1, count(k + 1));
    cp_async_commit();
    const bool live = lane < len_of(k);
    const size_t g0 = base + k * 32 + lane;
    float b[32];   // the tile's baseline, read while the copies are in flight: one memory latency per tile
#pragma unroll
    for (int j = 0; j < 32; ++j) b[j] = live && j < nr ? baseline[g0 + (size_t)j * T] : 0.0f;
    cp_async_wait<0>();
    __syncwarp();
    if (k == k0) convert(k0, len_of(k0));
    convert(k + 1, count(k + 1));
    __syncwarp();
    const int p = (int)(k & 1) * 32 + lane;
#pragma unroll
    for (int j0 = 0; j0 < 32; j0 += kNstepRows) {   // rows past nr are computed from stale tiles and never stored
      if (j0 >= nr) break;
      float acc[kNstepRows];
#pragma unroll
      for (int r = 0; r < kNstepRows; ++r) acc[r] = vv[j0 + r][(p + n) & 63];
#pragma unroll 2
      for (int i = n - 1; i >= 0; --i) {
        const int q = (p + i) & 63;
#pragma unroll
        for (int r = 0; r < kNstepRows; ++r) {
          const float2 x = rd[j0 + r][q];
          acc[r] = __fadd_rn(x.x, __fmul_rn(x.y, acc[r]));
        }
      }
#pragma unroll
      for (int r = 0; r < kNstepRows; ++r) {
        if (live && j0 + r < nr) {
          const size_t g = g0 + (size_t)(j0 + r) * T;
          ret[g] = acc[r];
          td[g] = __fsub_rn(acc[r], b[j0 + r]);
        }
      }
    }
    __syncwarp();   // slot k & 1 is reloaded by the next iteration's issue()
  }
}

// The pointer, size and overlap checks of a returns entry, in the header's order: NI inputs (the last one [N], the
// others [N, T]) then two [N, T] outputs, all fp32.  KTB_OK or KTB_ERR_ARG with the message set.
template <int NI>
static int check_buffers(const char* who, const void* const (&ptrs)[NI + 2], const char* const (&names)[NI + 2],
                         size_t N, size_t T) {
  for (int i = 0; i < NI + 2; ++i) {
    KTB_REQUIRE(ptrs[i] != nullptr, KTB_ERR_ARG, "%s: %s is NULL with N*T = %zu*%zu", who, names[i], N, T);
    KTB_REQUIRE(((uintptr_t)ptrs[i] & 3) == 0, KTB_ERR_ARG, "%s: %s is not 4-byte aligned", who, names[i]);
  }
  KTB_REQUIRE(T <= SIZE_MAX / 4 / N, KTB_ERR_ARG, "%s: N*T = %zu*%zu elements is too large", who, N, T);
  const size_t bytes = N * T * 4;
  for (int o = NI; o < NI + 2; ++o) {
    for (int i = 0; i < NI; ++i)
      KTB_REQUIRE(!overlaps(ptrs[o], bytes, ptrs[i], i == NI - 1 ? N * 4 : bytes), KTB_ERR_ARG, "%s: %s overlaps %s",
                  who, names[o], names[i]);
  }
  KTB_REQUIRE(!overlaps(ptrs[NI], bytes, ptrs[NI + 1], bytes), KTB_ERR_ARG, "%s: %s overlaps %s", who, names[NI],
              names[NI + 1]);
  KTB_REQUIRE((N + 31) / 32 <= 0x7fffffffULL, KTB_ERR_ARG, "%s: N = %zu rows is too many", who, N);
  return KTB_OK;
}

}  // namespace ktb

using namespace ktb;

extern "C" {

int ktb_gae_f32(int dev, const float* rewards, const float* values, const float* dones, const float* last_values,
                size_t N, size_t T, float gamma, float gamma_lam, float* adv, float* ret, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(std::isfinite(gamma) && std::isfinite(gamma_lam), KTB_ERR_ARG,
              "ktb_gae_f32: gamma (%g) and gamma_lam (%g) must be finite", (double)gamma, (double)gamma_lam);
  if (N == 0 || T == 0) return KTB_OK;
  if ((rc = check_buffers<4>("ktb_gae_f32", {rewards, values, dones, last_values, adv, ret},
                             {"rewards", "values", "dones", "last_values", "adv", "ret"}, N, T)))
    return rc;
  KTB_GUARD(dev);
  gae_kernel<<<(unsigned)((N + 31) / 32), 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      rewards, values, dones, last_values, N, T, gamma, gamma_lam, adv, ret);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int ktb_vtrace_f32(int dev, const float* log_rhos, const float* rewards, const float* values, const float* dones,
                   const float* bootstrap, size_t N, size_t T, float gamma, float lam, float rho_bar, float c_bar,
                   float pg_rho_bar, float* vs, float* pg_adv, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(std::isfinite(gamma) && std::isfinite(lam), KTB_ERR_ARG,
              "ktb_vtrace_f32: gamma (%g) and lam (%g) must be finite", (double)gamma, (double)lam);
  KTB_REQUIRE(rho_bar > 0.0f && c_bar > 0.0f && pg_rho_bar > 0.0f, KTB_ERR_ARG,
              "ktb_vtrace_f32: rho_bar (%g), c_bar (%g) and pg_rho_bar (%g) must be > 0 (+inf: no clip)",
              (double)rho_bar, (double)c_bar, (double)pg_rho_bar);
  if (N == 0 || T == 0) return KTB_OK;
  if ((rc = check_buffers<5>("ktb_vtrace_f32", {log_rhos, rewards, values, dones, bootstrap, vs, pg_adv},
                             {"log_rhos", "rewards", "values", "dones", "bootstrap", "vs", "pg_adv"}, N, T)))
    return rc;
  KTB_GUARD(dev);
  vtrace_kernel<<<(unsigned)((N + 31) / 32), 32, kVtraceSmem, reinterpret_cast<cudaStream_t>(stream)>>>(
      log_rhos, rewards, values, dones, bootstrap, N, T, gamma, lam, rho_bar, c_bar, pg_rho_bar, vs, pg_adv);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int ktb_retrace_f32(int dev, const float* log_rhos, const float* rewards, const float* q, const float* values,
                    const float* dones, const float* baseline, const float* bootstrap, size_t N, size_t T, float gamma,
                    float lam, float* ret, float* td, uintptr_t stream) {
  static std::atomic<unsigned> smem_set{0};   // the devices whose retrace_kernel has opted in to kRetraceSmem
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(std::isfinite(gamma) && std::isfinite(lam), KTB_ERR_ARG,
              "ktb_retrace_f32: gamma (%g) and lam (%g) must be finite", (double)gamma, (double)lam);
  if (N == 0 || T == 0) return KTB_OK;
  if ((rc = check_buffers<7>("ktb_retrace_f32", {log_rhos, rewards, q, values, dones, baseline, bootstrap, ret, td},
                             {"log_rhos", "rewards", "q", "values", "dones", "baseline", "bootstrap", "ret", "td"}, N,
                             T)))
    return rc;
  KTB_GUARD(dev);
  if (!(smem_set.load(std::memory_order_acquire) & (1u << dev))) {   // dev < kMaxDevices: require_device checked it
    KTB_CK(cudaFuncSetAttribute(retrace_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kRetraceSmem));
    smem_set.fetch_or(1u << dev, std::memory_order_release);
  }
  retrace_kernel<<<(unsigned)((N + 31) / 32), 32, kRetraceSmem, reinterpret_cast<cudaStream_t>(stream)>>>(
      log_rhos, rewards, q, values, dones, baseline, bootstrap, N, T, gamma, lam, ret, td);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int ktb_nstep_f32(int dev, const float* rewards, const float* values, const float* dones, const float* baseline,
                  const float* last_values, size_t N, size_t T, int n, float gamma, float* ret, float* td,
                  uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(n >= 1 && n <= 32, KTB_ERR_ARG, "ktb_nstep_f32: n = %d must be in [1, 32]", n);
  KTB_REQUIRE(std::isfinite(gamma), KTB_ERR_ARG, "ktb_nstep_f32: gamma (%g) must be finite", (double)gamma);
  if (N == 0 || T == 0) return KTB_OK;
  if ((rc = check_buffers<5>("ktb_nstep_f32", {rewards, values, dones, baseline, last_values, ret, td},
                             {"rewards", "values", "dones", "baseline", "last_values", "ret", "td"}, N, T)))
    return rc;
  KTB_GUARD(dev);
  const size_t n_tiles = (T + 31) / 32;
  size_t span = (n_tiles + 65534) / 65535;   // gridDim.y is at most 65535
  span = span > (size_t)kNstepSpan ? span : (size_t)kNstepSpan;
  const dim3 grid((unsigned)((N + 31) / 32), (unsigned)((n_tiles + span - 1) / span));
  nstep_kernel<<<grid, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(rewards, values, dones, baseline, last_values,
                                                                         N, T, n, gamma, span, ret, td);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

}  // extern "C"
