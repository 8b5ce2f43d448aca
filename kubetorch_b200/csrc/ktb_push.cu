// ktb_push.cu — the push/push form of scatter → exec → gather, synchronised INSIDE the kernels.
//
// ktb_scatter_map_gather (ktb_dispatch.cu) has every rank PULL its shard from the root (peer loads)
// and PUSH its result back (peer stores): one kernel per rank, but the rank's NVLink port then carries
// read requests + write data one way and read data + write acks the other.  Here both directions carry posted
// writes only:
//
//   root  : push_scatter_kernel  — ONE launch per call; CTAs run chunk-major: peer-STORE chunk c of every rank's
//           shard into that rank's staging buffer; the CTA that completes chunk c (per-chunk counter) publishes
//           ready[r][c] = seq (st.release.sys) in every rank's memory
//   rank r: push_consume_kernel  — ONE launch per call; the CTAs of chunk c spin (ld.acquire.sys, local memory)
//           until ready[c] >= seq, apply the op to the staged chunk (local HBM read) and peer-STORE the result into
//           the root's result arena; the last CTA publishes ack[r] = seq in the root's memory
//   root  : push_wait_kernel     — stream-ordered completion: spin until every ack[r] >= seq
//
// Why this shape: a GPU that drives both directions of its port (a kernel that loads from the peer and stores to it)
// sends read requests against its own write data; posted WRITES from each side need no round trip.  One kernel per
// chunk would drain the link at every launch boundary, so the chunk hand-off happens inside one resident grid per side.
//
// The flags replace host-side events, so the same code serves one controller process driving N GPUs
// and one process per GPU (CUDA IPC arenas): there is no host synchronisation on the data path at all.
// Staging is double-buffered by call parity; the root does not overwrite buffer (seq & 1) before the
// rank has acknowledged call seq-2.  Every spin carries a wall-clock timeout that raises a sticky
// status word instead of hanging the GPU.
//
// Replaces: kt/serving/spmd/spmd_supervisor.py:366-570 (fan-out, wait loop, concat) and
// kt/serving/remote_worker_pool.py:254-395 (per-pod POST + gather).
#include "ktb_common.cuh"

#include <algorithm>
#include <mutex>

namespace ktb {

constexpr int kPushMaxRanks = 16;
constexpr int kPushThreads = 256;
constexpr uint32_t kPushTile = 16384;          // bytes per CTA
struct PushScatterArgs {
  const uint8_t* src[kPushMaxRanks];             // root-local base of this rank's shard
  uint8_t* dst[kPushMaxRanks];                   // peer staging base (call-parity half already applied)
  unsigned long long shard_bytes[kPushMaxRanks];
  unsigned long long chunk_bytes[kPushMaxRanks]; // bytes per chunk of this rank's shard (same rule as the consumer)
  uint32_t tile_prefix[kPushMaxRanks + 1];       // tiles per chunk, prefix over ranks (identical for every chunk)
  unsigned long long* ready[kPushMaxRanks];      // peer: ready_r[0..n_chunks)
  const unsigned long long* ack[kPushMaxRanks];  // root-local: &ack[r]
  int n;
  int n_chunks;
  unsigned long long seq;
};

__global__ void __launch_bounds__(kPushThreads)
    push_scatter_kernel(const __grid_constant__ PushScatterArgs a, unsigned int* chunk_done, unsigned int* status) {
  const uint32_t tiles_per_chunk = a.tile_prefix[a.n];
  const uint32_t total_tiles = tiles_per_chunk * (uint32_t)a.n_chunks;
  __shared__ bool last;
  // CTAs walk the 16 KiB tiles in chunk-major order, one tile each unless the grid is capped, and report the tiles
  // of a chunk with ONE system fence + one atomic.  One tile per CTA measured best: many short-lived CTAs keep more
  // stores in flight than fewer CTAs streaming longer runs of tiles.
  uint32_t cur_chunk = 0xffffffffu, n_done = 0;
  auto flush = [&]() {   // all threads call it together
    __syncthreads();     // every thread's stores of the finished tiles are issued
    if (threadIdx.x == 0) {
      __threadfence_system();
      last = (atomicAdd(&chunk_done[cur_chunk], n_done) + n_done == tiles_per_chunk);
    }
    __syncthreads();
    if (last) {          // this CTA completed the chunk: publish "chunk landed" to every rank
      if (threadIdx.x < a.n) {
        __threadfence_system();
        st_release_sys(a.ready[threadIdx.x] + cur_chunk, a.seq);
      }
      if (threadIdx.x == 0) chunk_done[cur_chunk] = 0;
    }
    __syncthreads();     // `last` is reused
  };
  for (uint32_t tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const uint32_t c = tile / tiles_per_chunk;                // chunk 0 of every rank goes out first
    const uint32_t rem = tile % tiles_per_chunk;
    if (c != cur_chunk) {
      if (n_done) flush();
      cur_chunk = c;
      n_done = 0;
    }
    int seg = 0;
    while (seg + 1 < a.n && a.tile_prefix[seg + 1] <= rem) ++seg;
    // do not overwrite staging buffer (seq & 1) before the rank consumed call seq-2
    if (a.seq > 2) {
      if (threadIdx.x == 0) (void)spin_until(a.ack[seg], a.seq - 2, status);   // a timeout is recorded in *status
      __syncthreads();
    }
    const size_t shard = (size_t)a.shard_bytes[seg];
    const size_t cb = min(shard, (size_t)c * (size_t)a.chunk_bytes[seg]);
    const size_t ce = min(shard, cb + (size_t)a.chunk_bytes[seg]);
    const size_t off = cb + (size_t)(rem - a.tile_prefix[seg]) * kPushTile;
    if (off < ce) {
      const size_t len = (ce - off) < (size_t)kPushTile ? (ce - off) : (size_t)kPushTile;
      const uint8_t* s = a.src[seg] + off;
      uint8_t* d = a.dst[seg] + off;
      if (((((uintptr_t)s) | ((uintptr_t)d)) & 31) == 0) {
        const size_t nv = len >> 5;   // a full tile = 512 packets = 2 per thread, both loads first
        uint32_t w0[8], w1[8];
        const size_t v0 = threadIdx.x, v1 = threadIdx.x + kPushThreads;
        if (v0 < nv) ldg256_stream(s + (v0 << 5), w0);
        if (v1 < nv) ldg256_stream(s + (v1 << 5), w1);
        if (v0 < nv) stg256(d + (v0 << 5), w0);
        if (v1 < nv) stg256(d + (v1 << 5), w1);
        for (size_t e = (nv << 5) + threadIdx.x; e < len; e += kPushThreads) d[e] = s[e];
      } else {
        for (size_t e = threadIdx.x; e < len; e += kPushThreads) d[e] = s[e];
      }
    }
    ++n_done;
  }
  if (n_done) flush();
}

// Publish-only launch for calls with nothing to move (keeps the flag protocol uniform).
__global__ void push_publish_kernel(const __grid_constant__ PushScatterArgs a) {
  if (threadIdx.x < a.n)
    for (int c = 0; c < a.n_chunks; ++c) st_release_sys(a.ready[threadIdx.x] + c, a.seq);
}

template <int DT, int OP>
__global__ void __launch_bounds__(kPushThreads)
    push_consume_kernel(const uint8_t* stage, uint8_t* dst, size_t shard_bytes, size_t chunk_bytes,
                        uint32_t tiles_per_chunk, MapParams p,
                        const unsigned long long* ready, unsigned long long seq, unsigned long long* ack,
                        unsigned int* ticket, unsigned int* status) {
  constexpr size_t ES = dtype_size(DT);
  __shared__ bool flag;
  // One CTA per tile, tiles in increasing order = chunk order, and no tile loop: the kernel then keeps few registers
  // and many CTAs per SM (with a grid-stride loop it took 40 registers and 11 % longer on an H100 80GB HBM3 at 700 W).
  // One system fence per CTA before the ack ticket.
  const uint32_t tile = blockIdx.x;
  const uint32_t c = tile / tiles_per_chunk;
  const uint32_t t = tile % tiles_per_chunk;
  if (threadIdx.x == 0) flag = spin_until(ready + c, seq, status);
  __syncthreads();
  // the piece never arrived (the wait timed out and raised the sticky status word): do NOT map stale staging
  // data into the caller's result and do NOT acknowledge — the root's wait then times out too and the host maps
  // the status to PodTerminatedError; the session is torn down, so the unbalanced ticket does not matter
  if (!flag) return;
  const size_t cb = min(shard_bytes, (size_t)c * chunk_bytes);
  const size_t ce = min(shard_bytes, cb + chunk_bytes);
  const size_t off = cb + (size_t)t * kPushTile;
  if (off < ce) {
    const size_t len = (ce - off) < (size_t)kPushTile ? (ce - off) : (size_t)kPushTile;
    const uint8_t* s = stage + off;
    uint8_t* d = dst + off;
    if (((((uintptr_t)s) | ((uintptr_t)d)) & 31) == 0) {
      const size_t nv = len >> 5;
      uint32_t w0[8], w1[8];
      const size_t v0 = threadIdx.x, v1 = threadIdx.x + kPushThreads;
      if (v0 < nv) ldg256_stream(s + (v0 << 5), w0);
      if (v1 < nv) ldg256_stream(s + (v1 << 5), w1);
      if (v0 < nv) {
        apply_words<DT, OP, 8>(w0, p);
        stg256(d + (v0 << 5), w0);
      }
      if (v1 < nv) {
        apply_words<DT, OP, 8>(w1, p);
        stg256(d + (v1 << 5), w1);
      }
      const size_t tail = nv << 5;
      for (size_t e = threadIdx.x; e < (len - tail) / ES; e += kPushThreads)
        apply_elem<DT, OP>(s + tail + e * ES, d + tail + e * ES, p);
    } else {
      for (size_t e = threadIdx.x; e < len / ES; e += kPushThreads) apply_elem<DT, OP>(s + e * ES, d + e * ES, p);
    }
  }
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence_system();
    st_release_sys(ack, seq);   // results of the whole shard are in the root's memory
    *ticket = 0;
  }
}

__global__ void push_wait_kernel(const unsigned long long* ack, int n_ranks, int root_rank, unsigned long long seq,
                                 unsigned int* status) {
  const int r = threadIdx.x;
  if (r < n_ranks && r != root_rank) spin_until(&ack[r], seq, status);
}

// One flag per launch, stream-ordered: the copy-engine scatter's "rank consumed call seq-2" and "chunk landed", and the
// pushed MLP's "chunk c landed" and "this rank's call is done" (ktb_mlp.cu).
__global__ void flag_wait_kernel(const unsigned long long* flag, unsigned long long want, unsigned int* status) {
  if (threadIdx.x == 0) (void)spin_until(flag, want, status);
}
__global__ void flag_publish_kernel(unsigned long long* flag, unsigned long long seq) {
  if (threadIdx.x == 0) {
    __threadfence_system();
    st_release_sys(flag, seq);
  }
}

int launch_flag_wait(const unsigned long long* flag, unsigned long long want, unsigned int* status,
                     cudaStream_t stream) {
  flag_wait_kernel<<<1, 32, 0, stream>>>(flag, want, status);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int launch_flag_publish(unsigned long long* flag, unsigned long long seq, cudaStream_t stream) {
  flag_publish_kernel<<<1, 32, 0, stream>>>(flag, seq);
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

// Elements per chunk when a shard of shard_elems elements is cut into n_chunks pieces: ceil(shard / n_chunks) rounded
// up to 64 elements, at most the whole shard.  The root and the rank (possibly in different processes) both use it,
// so they agree on every chunk's bounds.
static size_t push_chunk_elems(size_t shard_elems, int n_chunks) {
  const size_t per = (shard_elems + (size_t)n_chunks - 1) / (size_t)n_chunks;
  return std::min(shard_elems, (per + 63) / 64 * 64);
}

// n_chunks of the chunk_elems form: as many pieces of exactly chunk_elems elements as the largest shard (rank 0's)
// needs, at least 1; any count past KTB_PUSH_MAX_CHUNKS comes back as KTB_PUSH_MAX_CHUNKS + 1 for the caller to reject.
static int push_chunk_count(size_t n_elems, size_t granule, int n_ranks, size_t chunk_elems) {
  size_t b0 = 0, e0 = 0;
  ktb_shard_bounds(n_elems / granule, n_ranks, 0, &b0, &e0);
  const size_t n = std::max<size_t>(1, ((e0 - b0) * granule + chunk_elems - 1) / chunk_elems);
  return (int)std::min<size_t>(n, KTB_PUSH_MAX_CHUNKS + 1);
}

// The argument checks of the root side that the SM form (push_scatter_impl) and the copy-engine form share.
static int check_push_scatter(const char* who, int root_dev, const void* src_root, size_t n_elems, size_t granule,
                              int dtype, int n_ranks, int root_rank, void* const* stage_peer, size_t stage_stride,
                              void* const* ctrl_peer, const void* ctrl_root, unsigned long long seq) {
  int rc = require_device(root_dev);
  if (rc) return rc;
  rc = check_dtype(who, dtype);
  if (rc) return rc;
  KTB_REQUIRE(n_ranks > 0 && n_ranks <= kPushMaxRanks && root_rank >= 0 && root_rank < n_ranks, KTB_ERR_ARG,
              "%s: bad ranks %d/%d", who, root_rank, n_ranks);
  KTB_REQUIRE(src_root && stage_peer && ctrl_peer && ctrl_root && seq > 0, KTB_ERR_ARG, "%s: null argument", who);
  KTB_REQUIRE(granule > 0 && n_elems % granule == 0, KTB_ERR_ARG, "%s: n_elems not a multiple of granule", who);
  for (int r = 0; r < n_ranks; ++r) {
    if (r == root_rank || !stage_peer[r]) continue;   // null staging = rank served by another scatter call
    size_t b = 0, e = 0;
    ktb_shard_bounds(n_elems / granule, n_ranks, r, &b, &e);
    KTB_REQUIRE(ctrl_peer[r], KTB_ERR_ARG, "%s: rank %d has no control block", who, r);
    KTB_REQUIRE((e - b) * granule * dtype_size(dtype) <= stage_stride, KTB_ERR_ARG,
                "%s: shard of rank %d exceeds stage_stride", who, r);
  }
  return KTB_OK;
}

}  // namespace ktb

using namespace ktb;

extern "C" {

size_t ktb_push_control_bytes(void) { return 4096; }

// (control-block layout: KTB_CTRL_* in ktb_common.cuh)

// chunk_elems == 0: n_chunks pieces per shard (push_chunk_elems); otherwise pieces of exactly chunk_elems elements
// (the consumer of ktb_mlp_bf16_pushed wants whole GEMM row chunks), n_chunks = ceil(largest shard / chunk_elems).
static int push_scatter_impl(const char* who, int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype,
                             int n_ranks, int root_rank, void* const* stage_peer, size_t stage_stride,
                             void* const* ctrl_peer, void* ctrl_root, int n_chunks, size_t chunk_elems,
                             unsigned long long seq, int ctas_per_sm, uintptr_t stream) {
  int rc = check_push_scatter(who, root_dev, src_root, n_elems, granule, dtype, n_ranks, root_rank, stage_peer,
                              stage_stride, ctrl_peer, ctrl_root, seq);
  if (rc) return rc;
  if (chunk_elems) n_chunks = push_chunk_count(n_elems, granule, n_ranks, chunk_elems);
  KTB_REQUIRE(n_chunks > 0 && n_chunks <= KTB_PUSH_MAX_CHUNKS, KTB_ERR_ARG, "%s: n_chunks %d out of range", who, n_chunks);
  const size_t es = dtype_size(dtype);
  KTB_GUARD(root_dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* croot = static_cast<uint8_t*>(ctrl_root);
  // per call parity: the scatters of two consecutive calls may overlap when the caller alternates streams
  unsigned int* chunk_done =
      reinterpret_cast<unsigned int*>(croot + KTB_CTRL_CHUNK_DONE) + (size_t)(seq & 1) * KTB_PUSH_MAX_CHUNKS;
  unsigned int* status = reinterpret_cast<unsigned int*>(croot + KTB_CTRL_STATUS);
  const size_t buf_off = (size_t)(seq & 1) * stage_stride;
  PushScatterArgs a;
  a.n = 0;
  a.n_chunks = n_chunks;
  a.seq = seq;
  a.tile_prefix[0] = 0;
  for (int r = 0; r < n_ranks; ++r) {
    // a null stage_peer[r]: not served by this call (a hybrid scatter splits the ranks between two engines)
    if (r == root_rank || !stage_peer[r]) continue;
    size_t sb = 0, se = 0;
    ktb_shard_bounds(n_elems / granule, n_ranks, r, &sb, &se);
    sb *= granule;
    se *= granule;
    const size_t per = chunk_elems ? chunk_elems : push_chunk_elems(se - sb, n_chunks);
    const int i = a.n++;
    a.src[i] = static_cast<const uint8_t*>(src_root) + sb * es;
    a.dst[i] = static_cast<uint8_t*>(stage_peer[r]) + buf_off;
    a.shard_bytes[i] = (se - sb) * es;
    a.chunk_bytes[i] = per * es;
    a.tile_prefix[i + 1] = a.tile_prefix[i] + (uint32_t)((per * es + kPushTile - 1) / kPushTile);
    a.ready[i] = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ctrl_peer[r]) + KTB_CTRL_READY);
    a.ack[i] = reinterpret_cast<const unsigned long long*>(croot + KTB_CTRL_ACK) + r;
  }
  if (a.n == 0) return KTB_OK;
  const uint32_t tiles_per_chunk = a.tile_prefix[a.n];
  if (tiles_per_chunk == 0) {
    push_publish_kernel<<<1, 32, 0, st>>>(a);
  } else {
    // ctas_per_sm <= 0: no cap, one CTA per tile.  Caps measured slower for the element-wise call;
    // ktb_push_scatter_chunked passes its own cap for the MLP.
    const size_t total = (size_t)tiles_per_chunk * (size_t)n_chunks;
    const size_t cap = ctas_per_sm > 0 ? (size_t)device_info(root_dev)->sm_count * (size_t)ctas_per_sm : total;
    push_scatter_kernel<<<(unsigned)std::min(total, cap), kPushThreads, 0, st>>>(a, chunk_done, status);
  }
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

int ktb_push_scatter(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype, int n_ranks,
                     int root_rank, void* const* stage_peer, size_t stage_stride, void* const* ctrl_peer,
                     void* ctrl_root, int n_chunks, unsigned long long seq, uintptr_t stream) {
  return push_scatter_impl("ktb_push_scatter", root_dev, src_root, n_elems, granule, dtype, n_ranks, root_rank, stage_peer,
                           stage_stride, ctrl_peer, ctrl_root, n_chunks, 0, seq, 0, stream);
}

int ktb_push_scatter_chunked(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype, int n_ranks,
                             int root_rank, void* const* stage_peer, size_t stage_stride, void* const* ctrl_peer,
                             void* ctrl_root, size_t chunk_elems, int ctas_per_sm, unsigned long long seq,
                             uintptr_t stream) {
  KTB_REQUIRE(chunk_elems > 0, KTB_ERR_ARG, "ktb_push_scatter_chunked: chunk_elems must be positive");
  return push_scatter_impl("ktb_push_scatter_chunked", root_dev, src_root, n_elems, granule, dtype, n_ranks, root_rank,
                           stage_peer, stage_stride, ctrl_peer, ctrl_root, 0, chunk_elems, seq, ctas_per_sm, stream);
}

// ---- copy-engine form of the root side: no SM of the root is used ------------------------------------------------
// With n_sides (0 to 2; anything else, or null sides, is KTB_ERR_ARG) side sources (PushSide, a shard row being
// `granule` elements), each rides along chunk by chunk beside the rows and behind the same ack wait, with ready[c]
// published after every copy of chunk c.  Their checks come after every check of the plain form: per side in order a
// null source, then row_bytes and whole-row chunks, then per served rank its regions (check_push_sides).
static int push_scatter_ce_impl(const char* who, int root_dev, const void* src_root, size_t n_elems, size_t granule,
                                int dtype, int n_ranks, int root_rank, const int* devs, void* const* stage_peer,
                                size_t stage_stride, void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems,
                                int n_sides, const PushSide* sides, unsigned long long seq, uintptr_t stream) {
  int rc = check_push_scatter(who, root_dev, src_root, n_elems, granule, dtype, n_ranks, root_rank, stage_peer,
                              stage_stride, ctrl_peer, ctrl_root, seq);
  if (rc) return rc;
  KTB_REQUIRE(devs && chunk_elems > 0, KTB_ERR_ARG, "%s: null devs or zero chunk_elems", who);
  const int n_chunks = push_chunk_count(n_elems, granule, n_ranks, chunk_elems);
  KTB_REQUIRE(n_chunks <= KTB_PUSH_MAX_CHUNKS, KTB_ERR_ARG, "%s: more than %d chunks", who, KTB_PUSH_MAX_CHUNKS);
  const size_t es = dtype_size(dtype);
  KTB_REQUIRE(n_sides >= 0 && n_sides <= 2 && (n_sides == 0 || sides), KTB_ERR_ARG,
              "%s: 1 or 2 side sources, with non-null arrays", who);
  for (int k = 0; k < n_sides; ++k) {
    const PushSide& sd = sides[k];
    KTB_REQUIRE(sd.src || n_elems == 0, KTB_ERR_ARG, "%s: null %s", who, sd.name);
    KTB_REQUIRE(sd.row_bytes > 0 && chunk_elems % granule == 0, KTB_ERR_ARG,
                "%s: row_bytes must be positive and chunk_elems whole rows", who);
  }
  for (int r = 0; n_sides > 0 && r < n_ranks; ++r) {
    if (r == root_rank || !stage_peer[r]) continue;
    size_t b = 0, e = 0;
    ktb_shard_bounds(n_elems / granule, n_ranks, r, &b, &e);
    rc = check_push_sides(who, sides, n_sides, e - b, granule * es, stage_stride);
    if (rc) return rc;
  }
  KTB_GUARD(root_dev);
  // one library stream (and fork/join event pair) per destination rank on the root device, created on first use:
  // every peer's copies ride their own copy-engine queue, chunk-major issue order
  static std::mutex mu;
  static cudaStream_t ce_stream[kMaxDevices][kPushMaxRanks] = {};
  static cudaEvent_t ce_done[kMaxDevices][kPushMaxRanks] = {};
  static cudaEvent_t ce_start[kMaxDevices] = {};
  std::lock_guard<std::mutex> lk(mu);   // also serialises concurrent CE scatters of one root (they share the streams)
  if (!ce_start[root_dev]) KTB_CK(cudaEventCreateWithFlags(&ce_start[root_dev], cudaEventDisableTiming));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* croot = static_cast<uint8_t*>(ctrl_root);
  unsigned int* status = reinterpret_cast<unsigned int*>(croot + KTB_CTRL_STATUS);
  const size_t buf_off = (size_t)(seq & 1) * stage_stride;
  KTB_CK(cudaEventRecord(ce_start[root_dev], st));   // the observations are ready once prior work on `st` is done
  size_t sb[kPushMaxRanks], sl[kPushMaxRanks];
  for (int r = 0; r < n_ranks; ++r) {
    size_t b = 0, e = 0;
    ktb_shard_bounds(n_elems / granule, n_ranks, r, &b, &e);
    sb[r] = b * granule;
    sl[r] = (e - b) * granule;
    if (r == root_rank || !stage_peer[r]) continue;   // null staging = rank served by another scatter call
    if (!ce_stream[root_dev][r]) {
      KTB_CK(cudaStreamCreateWithFlags(&ce_stream[root_dev][r], cudaStreamNonBlocking));
      KTB_CK(cudaEventCreateWithFlags(&ce_done[root_dev][r], cudaEventDisableTiming));
    }
    KTB_CK(cudaStreamWaitEvent(ce_stream[root_dev][r], ce_start[root_dev], 0));
    if (seq > 2) {   // do not overwrite staging half (seq & 1) before the rank consumed call seq-2
      rc = launch_flag_wait(reinterpret_cast<const unsigned long long*>(croot + KTB_CTRL_ACK) + r, seq - 2, status,
                            ce_stream[root_dev][r]);
      if (rc) return rc;
    }
  }
  for (size_t c = 0; c < (size_t)n_chunks; ++c) {
    for (int r = 0; r < n_ranks; ++r) {
      if (r == root_rank || !stage_peer[r]) continue;
      cudaStream_t cs = ce_stream[root_dev][r];
      const size_t lo = std::min(sl[r], c * chunk_elems), hi = std::min(sl[r], lo + chunk_elems);
      if (hi > lo)
        KTB_CK(cudaMemcpyPeerAsync(static_cast<uint8_t*>(stage_peer[r]) + buf_off + lo * es, devs[r],
                                   static_cast<const uint8_t*>(src_root) + (sb[r] + lo) * es, root_dev, (hi - lo) * es, cs));
      for (int k = 0; k < n_sides && hi > lo; ++k)   // the same rows' side sources, beside them
        KTB_CK(cudaMemcpyPeerAsync(
            static_cast<uint8_t*>(stage_peer[r]) + buf_off + sides[k].offset + lo / granule * sides[k].row_bytes,
            devs[r], static_cast<const uint8_t*>(sides[k].src) + (sb[r] + lo) / granule * sides[k].row_bytes,
            root_dev, (hi - lo) / granule * sides[k].row_bytes, cs));
      unsigned long long* ready =
          reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ctrl_peer[r]) + KTB_CTRL_READY) + c;
      rc = launch_flag_publish(ready, seq, cs);   // stream-ordered behind the copy
      if (rc) return rc;
    }
  }
  for (int r = 0; r < n_ranks; ++r) {   // the caller's stream "contains" the scatter (src may be reused after it)
    if (r == root_rank || !stage_peer[r]) continue;
    KTB_CK(cudaEventRecord(ce_done[root_dev][r], ce_stream[root_dev][r]));
    KTB_CK(cudaStreamWaitEvent(st, ce_done[root_dev][r], 0));
  }
  return KTB_OK;
}

int ktb_push_scatter_ce(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype, int n_ranks,
                        int root_rank, const int* devs, void* const* stage_peer, size_t stage_stride,
                        void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems, unsigned long long seq,
                        uintptr_t stream) {
  return push_scatter_ce_impl("ktb_push_scatter_ce", root_dev, src_root, n_elems, granule, dtype, n_ranks, root_rank,
                              devs, stage_peer, stage_stride, ctrl_peer, ctrl_root, chunk_elems, 0, nullptr, seq,
                              stream);
}

int ktb_push_scatter_ce_masked(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype,
                               int n_ranks, int root_rank, const int* devs, void* const* stage_peer,
                               size_t stage_stride, void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems,
                               const void* mask_root, size_t row_bytes, size_t mask_offset, unsigned long long seq,
                               uintptr_t stream) {
  const PushSide side{mask_root, row_bytes, mask_offset, 1, "mask"};
  return push_scatter_ce_impl("ktb_push_scatter_ce_masked", root_dev, src_root, n_elems, granule, dtype, n_ranks,
                              root_rank, devs, stage_peer, stage_stride, ctrl_peer, ctrl_root, chunk_elems, 1, &side,
                              seq, stream);
}

int ktb_push_scatter_ce_sides(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype,
                              int n_ranks, int root_rank, const int* devs, void* const* stage_peer, size_t stage_stride,
                              void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems, int n_sides,
                              const void* const* side_src, const size_t* side_row_bytes, const size_t* side_offset,
                              unsigned long long seq, uintptr_t stream) {
  static const char* const kNames[2] = {"side 0", "side 1"};
  // a bad count or null arrays reach the impl as no sides at all, which it refuses after the plain form's checks
  const bool ok = n_sides >= 1 && n_sides <= 2 && side_src && side_row_bytes && side_offset;
  PushSide sides[2];
  for (int k = 0; ok && k < n_sides; ++k) sides[k] = {side_src[k], side_row_bytes[k], side_offset[k], 1, kNames[k]};
  return push_scatter_ce_impl("ktb_push_scatter_ce_sides", root_dev, src_root, n_elems, granule, dtype, n_ranks,
                              root_rank, devs, stage_peer, stage_stride, ctrl_peer, ctrl_root, chunk_elems,
                              ok ? n_sides : -1, ok ? sides : nullptr, seq, stream);
}

int ktb_push_consume(int dev, int op, int dtype, const void* stage_local, size_t stage_stride, void* dst_root_shard,
                     size_t shard_elems, double alpha, double beta, void* ctrl_local, void* ctrl_root_peer, int rank,
                     int n_chunks, unsigned long long seq, uintptr_t stream) {
  int rc = require_device(dev);
  if (rc) return rc;
  rc = check_elementwise("ktb_push_consume", op, dtype);
  if (rc) return rc;
  KTB_REQUIRE(n_chunks > 0 && n_chunks <= KTB_PUSH_MAX_CHUNKS && rank >= 0 && rank < kPushMaxRanks && seq > 0, KTB_ERR_ARG,
              "ktb_push_consume: bad chunk/rank arguments");
  KTB_REQUIRE(stage_local && ctrl_local && ctrl_root_peer && (dst_root_shard || shard_elems == 0), KTB_ERR_ARG,
              "ktb_push_consume: null argument");
  KTB_GUARD(dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const MapParams p = make_params(alpha, beta, dtype);
  uint8_t* cl = static_cast<uint8_t*>(ctrl_local);
  const unsigned long long* ready = reinterpret_cast<const unsigned long long*>(cl + KTB_CTRL_READY);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(cl + KTB_CTRL_TICKET);
  unsigned int* status = reinterpret_cast<unsigned int*>(cl + KTB_CTRL_STATUS);
  unsigned long long* ack =
      reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ctrl_root_peer) + KTB_CTRL_ACK) + rank;
  const uint8_t* stage = static_cast<const uint8_t*>(stage_local) + (size_t)(seq & 1) * stage_stride;
  const size_t es = dtype_size(dtype);
  const size_t chunk_bytes = push_chunk_elems(shard_elems, n_chunks) * es, shard_bytes = shard_elems * es;
  const uint32_t tpc = (uint32_t)std::max<size_t>(1, (chunk_bytes + kPushTile - 1) / kPushTile);
  const unsigned grid = (unsigned)((size_t)tpc * (size_t)n_chunks);   // one CTA per tile
  uint8_t* d = static_cast<uint8_t*>(dst_root_shard);
  return dispatch_elementwise(op, dtype, [&](auto dt, auto o) {
    push_consume_kernel<dt, o><<<grid, kPushThreads, 0, st>>>(stage, d, shard_bytes, chunk_bytes, tpc, p, ready, seq,
                                                              ack, ticket, status);
    KTB_CK(cudaGetLastError());
    return KTB_OK;
  });
}

int ktb_push_wait(int root_dev, void* ctrl_root, int n_ranks, int root_rank, unsigned long long seq, uintptr_t stream) {
  int rc = require_device(root_dev);
  if (rc) return rc;
  KTB_REQUIRE(ctrl_root && n_ranks > 0 && n_ranks <= kPushMaxRanks, KTB_ERR_ARG, "ktb_push_wait: bad arguments");
  KTB_GUARD(root_dev);
  uint8_t* croot = static_cast<uint8_t*>(ctrl_root);
  push_wait_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const unsigned long long*>(croot + KTB_CTRL_ACK), n_ranks, root_rank, seq,
      reinterpret_cast<unsigned int*>(croot + KTB_CTRL_STATUS));
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

// Reads (synchronously) the sticky timeout status of a control block: 0 = healthy.
int ktb_push_status(int dev, const void* ctrl, unsigned int* out) {
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_REQUIRE(ctrl && out, KTB_ERR_ARG, "ktb_push_status: null argument");
  KTB_GUARD(dev);
  KTB_CK(cudaMemcpy(out, static_cast<const uint8_t*>(ctrl) + KTB_CTRL_STATUS, sizeof(unsigned int),
                    cudaMemcpyDeviceToHost));
  return KTB_OK;
}

}  // extern "C"
