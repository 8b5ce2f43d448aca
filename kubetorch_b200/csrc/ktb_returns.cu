// ktb_returns.cu — generalized advantage estimation (ktb_gae_f32): PPO's advantages and λ-returns of env-major
// [N, T] rollouts, the reverse linear recurrence of include/ktb200.h evaluated exactly as written there.
//
// HBM-bound: 20·N·T + 4·N bytes, a handful of flops per element.  The recurrence runs along a row, but the rows are
// stored env-major, so one thread per row would read with a stride of T elements.  Instead each warp owns 32 rows
// and walks T backwards in 32-step tiles:
//   loads  for each of its rows the 32 lanes copy 32 consecutive steps of rewards, values and dones into shared
//          tiles (cp.async, 4 bytes per lane: any T and any 4-byte alignment take the same path, and each row's
//          32 words are one coalesced access), rows padded to 33 words so that the scan's column reads hit 32 banks;
//   scan   lane i runs row i's recurrence over the tile, right to left, with __fadd_rn / __fmul_rn / __fsub_rn so that
//          nothing is contracted into an FMA, and writes adv over the rewards and ret over the values;
//   stores the lanes write the tile's rows of adv and ret back as consecutive steps.
// kStages tiles are in flight per warp: the loads of the next two (earlier) tiles are issued before the current one
// is scanned.  A tile shorter than 32 steps (T % 32 at the end of the row, or T < 32) is copied by flat index over
// its rows, so that small T still moves whole segments.
#include "ktb_common.cuh"

#include <cmath>

namespace ktb {

constexpr int kGaeStages = 3;   // 3 x 12.4 KiB of shared tiles per warp
constexpr int kGaePad = 33;

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

// One warp per block and per 32 rows.
__global__ void __launch_bounds__(32)
    gae_kernel(const float* __restrict__ rewards, const float* __restrict__ values, const float* __restrict__ dones,
               const float* __restrict__ last_values, size_t N, size_t T, float gamma, float gamma_lam,
               float* __restrict__ adv, float* __restrict__ ret) {
  __shared__ float tile[kGaeStages][3][32][kGaePad];   // [stage][rewards → adv, values → ret, dones][row][step]
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
      float(*s)[32][kGaePad] = tile[k % kGaeStages];
      for_tile(nr, len_of(t0), lane, [&](int j, int c) {
        const size_t g = base + (size_t)j * T + t0 + c;
        cp_async4(&s[0][j][c], rewards + g);
        cp_async4(&s[1][j][c], values + g);
        cp_async4(&s[2][j][c], dones + g);
      });
    }
    cp_async_commit();   // one group per tile, empty past the first step: wait_group counts stay uniform
  };

  for (int k = 0; k < kGaeStages - 1; ++k) issue(k);
  float acc = 0.0f;
  float nv = lane < nr ? last_values[row0 + lane] : 0.0f;
  for (size_t k = 0; k < n_tiles; ++k) {
    issue(k + kGaeStages - 1);
    cp_async_wait<kGaeStages - 1>();   // this lane's copies of tile k have landed
    __syncwarp();                      // ... and every other lane's
    float(*s)[32][kGaePad] = tile[k % kGaeStages];
    const size_t t0 = t0_of(k);
    const int len = len_of(t0);
    if (lane < nr) {
      float* rw = s[0][lane];
      float* vl = s[1][lane];
      const float* dn = s[2][lane];
      for (int c = len - 1; c >= 0; --c) {
        const float v = vl[c];
        const float nt = __fsub_rn(1.0f, dn[c]);
        const float delta = __fsub_rn(__fadd_rn(rw[c], __fmul_rn(__fmul_rn(gamma, nv), nt)), v);
        acc = __fadd_rn(delta, __fmul_rn(__fmul_rn(gamma_lam, nt), acc));
        rw[c] = acc;
        vl[c] = __fadd_rn(acc, v);
        nv = v;
      }
    }
    __syncwarp();
    for_tile(nr, len, lane, [&](int j, int c) {
      const size_t g = base + (size_t)j * T + t0 + c;
      adv[g] = s[0][j][c];
      ret[g] = s[1][j][c];
    });
    __syncwarp();   // the stage is reloaded by the next iteration's issue()
  }
}

static bool overlaps(const void* a, size_t an, const void* b, size_t bn) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + bn && y < x + an;
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
  const void* ptrs[6] = {rewards, values, dones, last_values, adv, ret};
  const char* names[6] = {"rewards", "values", "dones", "last_values", "adv", "ret"};
  for (int i = 0; i < 6; ++i) {
    KTB_REQUIRE(ptrs[i] != nullptr, KTB_ERR_ARG, "ktb_gae_f32: %s is NULL with N*T = %zu*%zu", names[i], N, T);
    KTB_REQUIRE(((uintptr_t)ptrs[i] & 3) == 0, KTB_ERR_ARG, "ktb_gae_f32: %s is not 4-byte aligned", names[i]);
  }
  KTB_REQUIRE(T <= SIZE_MAX / 4 / N, KTB_ERR_ARG, "ktb_gae_f32: N*T = %zu*%zu elements is too large", N, T);
  const size_t bytes = N * T * 4;
  const size_t in_bytes[4] = {bytes, bytes, bytes, N * 4};
  for (int o = 4; o < 6; ++o) {
    for (int i = 0; i < 4; ++i)
      KTB_REQUIRE(!overlaps(ptrs[o], bytes, ptrs[i], in_bytes[i]), KTB_ERR_ARG, "ktb_gae_f32: %s overlaps %s",
                  names[o], names[i]);
  }
  KTB_REQUIRE(!overlaps(adv, bytes, ret, bytes), KTB_ERR_ARG, "ktb_gae_f32: adv overlaps ret");
  KTB_GUARD(dev);
  const size_t grid = (N + 31) / 32;
  KTB_REQUIRE(grid <= 0x7fffffffULL, KTB_ERR_ARG, "ktb_gae_f32: N = %zu rows is too many", N);
  gae_kernel<<<(unsigned)grid, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(rewards, values, dones, last_values,
                                                                                   N, T, gamma, gamma_lam, adv, ret);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

}  // extern "C"
