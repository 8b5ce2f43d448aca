/*
 * ktb200.h — C-ABI of libktb200.so, the H100 (sm_90a) dispatch backend for
 * kubetorch's data-parallel remote-call path.
 *
 * The reference (run-house/kubetorch @ 96fac95, python_client/kubetorch, "kt/"
 * below) has no FFI: its hot path is CPython pickle/base64/JSON + HTTP +
 * multiprocessing.Queue.  Every entry point here therefore cites the reference
 * *Python* function whose work it replaces on this route (SURVEY.md §8(a)/(b)):
 *
 *   pack / unpack          kt/serving/utils.py:730-749 (_serialize_body: pickle+b64 of args)
 *                          kt/serving/http_server.py:1768-1822 (_parse_callable_params: b64decode+unpickle)
 *                          kt/serving/http_server.py:1825-1842 (_serialize_result)
 *                          kt/serving/utils.py:787-813 (_deserialize_response)
 *   broadcast / scatter    kt/serving/spmd/spmd_supervisor.py:341,439-455 (params_list=[params]*P → call_all)
 *                          kt/serving/process_pool.py:125-212 (mp.Queue.put per rank)
 *                          kt/serving/remote_worker_pool.py:254-316 (HTTP POST per pod)
 *   map (exec)             kt/serving/http_server.py:1845-1891 (execute_callable_async → user fn)
 *   gather / gather-reduce kt/serving/spmd/spmd_supervisor.py:547-570 (local_responses + worker_responses)
 *                          kt/serving/process_pool.py:214-234 (_response_router)
 *   shard bounds           user-side `x.chunk(WORLD_SIZE)[RANK]` driven by the env contract of
 *                          kt/serving/process_worker.py:75-102
 *
 * Conventions
 *   - All functions return 0 on success, a negative ktb_status on failure; the
 *     message is available from ktb_last_error() (thread-local).
 *   - Buffers are caller-owned (PyTorch tensors: tensor.data_ptr()); the library
 *     borrows them for the duration of the enqueued work and never frees them.
 *     Memory from ktb_arena_alloc / ktb_host_alloc is library-owned until the
 *     matching free or ktb_shutdown.
 *   - `stream` is a cudaStream_t passed as uintptr_t (0 = legacy default stream).
 *     Calls enqueue and return without a host sync unless stated otherwise.
 *   - Device pointers may be local, peer-mapped (NVLink P2P / CUDA IPC) or
 *     mapped pinned host memory; the kernels only require what each entry states.
 *   - Thread-safe. No torch types cross this boundary.
 */
#ifndef KTB200_H
#define KTB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KTB_VERSION 100 /* 0.1.0 */

typedef enum {
  KTB_OK = 0,
  KTB_ERR_CUDA = -1,     /* a CUDA runtime call failed; see ktb_last_error() */
  KTB_ERR_ARG = -2,      /* invalid argument (null pointer, bad enum, misaligned, too large) */
  KTB_ERR_STATE = -3,    /* library not initialised / device not registered */
  KTB_ERR_UNSUPPORTED = -4
} ktb_status;

/* Mapped-callable vocabulary: the closed set of user callables that run as kernels. */
typedef enum {
  KTB_OP_IDENTITY = 0,   /* y = x                         (BASELINE config C5)       */
  KTB_OP_SCALE = 1,      /* y = x * alpha                 (BASELINE config C2: x→2x) */
  KTB_OP_AFFINE = 2      /* y = (x * alpha) + beta, each step rounded to dtype; for BF16/F16 beta is
                          * itself rounded to the dtype first (torch CPU eager scalar semantics)  */
} ktb_op;

typedef enum {
  KTB_U8 = 0,            /* raw bytes; identity only */
  KTB_F32 = 1,
  KTB_BF16 = 2,
  KTB_I32 = 3,           /* wrapping two's-complement arithmetic (torch semantics) */
  KTB_I64 = 4,
  KTB_F16 = 5            /* op-math in fp32, rounded to half (RNE) after each step, like ATen */
} ktb_dtype;

/* Kernel variant selector for the element-wise map (all bit-identical in output). */
typedef enum {
  KTB_VARIANT_AUTO = 0,  /* widest vector path the pointers allow */
  KTB_VARIANT_VEC = 1,   /* register path: 256-/128-bit LDG/STG, unrolled, persistent grid */
  KTB_VARIANT_TMA = 2,   /* cp.async.bulk global→shared ring, compute in shared, bulk store */
  KTB_VARIANT_SCALAR = 3 /* element-at-a-time (any alignment) */
} ktb_variant;

/* ---- runtime -------------------------------------------------------------------------- */

/* Register devices dev_ids[0..n_dev) with the library and enable peer access between every
 * ordered pair that supports it.  Replaces the rendezvous of kt/serving/distributed_supervisor.py:90-174
 * (pod_ips quorum) by a static local membership.  Idempotent; devices accumulate across calls. */
int ktb_init(int n_dev, const int* dev_ids);
int ktb_shutdown(void);
const char* ktb_last_error(void);
int ktb_version(void);
/* Number of SMs of a registered device (132 on H100 SXM), or a negative status. */
int ktb_sm_count(int dev);
/* 1 if `dev` can read/write `peer` memory directly (after ktb_init), else 0; negative on error. */
int ktb_peer_enabled(int dev, int peer);

/* ---- arenas: library-owned memory (cudaMalloc / cudaHostAlloc), IPC-exportable ----------- */

int ktb_arena_alloc(int dev, size_t nbytes, void** out);
int ktb_arena_free(int dev, void* ptr);
/* Pinned, device-mapped host memory (portable across registered devices). */
int ktb_host_alloc(size_t nbytes, void** out);
int ktb_host_free(void* ptr);
/* NUMA node of a registered device (sysfs, via its PCI bus id), or -1 if unknown. */
int ktb_device_numa_node(int dev);
/* Pinned host block whose byte range (part_end[i-1], part_end[i]] is FIRST-TOUCHED on the NUMA node of
 * device part_dev[i] (by that device's issue thread) before the block is page-locked (cudaHostRegister,
 * portable + mapped), so shard i's DMA never crosses the socket interconnect.  n_parts == 0 → plain block.
 * Replaces the client-side argument/result buffers of kt/serving/http_client.py:1041-1111. */
int ktb_host_alloc_sharded(size_t nbytes, int n_parts, const size_t* part_end, const int* part_dev, void** out);
int ktb_host_free_sharded(void* ptr);
/* CUDA IPC for process-per-rank workers (the reference's ProcessWorker model,
 * kt/serving/process_worker.py:15-60).  `ptr` must be the base of a ktb_arena_alloc block. */
#define KTB_IPC_HANDLE_BYTES 64
int ktb_ipc_export(int dev, void* ptr, unsigned char handle[KTB_IPC_HANDLE_BYTES]);
int ktb_ipc_open(int dev, const unsigned char handle[KTB_IPC_HANDLE_BYTES], void** out);
int ktb_ipc_close(int dev, void* ptr);

/* ---- shard partition ------------------------------------------------------------------- */

/* Bounds [begin,end) in elements of rank `rank`'s shard of an n-element dim-0 split over
 * `world` ranks, following torch.chunk: chunk = ceil(n/world); ranks past the data get an
 * empty shard (begin == end == n).  This is what the reference's user functions compute
 * from RANK/WORLD_SIZE (`x.chunk(w)[r]`, SURVEY.md Appendix A). */
int ktb_shard_bounds(size_t n, int world, int rank, size_t* begin, size_t* end);

/* ---- element-wise map: "execute the mapped callable" -------------------------------------- */

/* dst[i] = op(src[i]) for i in [0, n_elems).  src/dst may be local, peer or mapped-host
 * pointers valid on `dev`; they must be element-aligned and must not partially overlap
 * (src == dst is allowed).  alpha/beta are converted to the dtype's op-math type
 * (float for F32/BF16, int64 for I32/I64).  KTB_U8 supports KTB_OP_IDENTITY only.
 * KTB_VARIANT_TMA / _VEC need 16-byte aligned src and dst and silently use the next narrower
 * path otherwise (all variants are bit-identical). */
int ktb_map(int dev, int op, int dtype, const void* src, void* dst, size_t n_elems,
            double alpha, double beta, int variant, uintptr_t stream);

/* Named wrappers (SURVEY.md §8(b) B4 naming). */
int ktb_map_identity_u8(int dev, const void* src, void* dst, size_t nbytes, uintptr_t stream);
int ktb_map_scale_f32(int dev, const float* src, float* dst, size_t n, float alpha, uintptr_t stream);
int ktb_map_affine_f32(int dev, const float* src, float* dst, size_t n, float alpha, float beta, uintptr_t stream);
int ktb_map_scale_bf16(int dev, const void* src, void* dst, size_t n, float alpha, uintptr_t stream);
int ktb_map_affine_bf16(int dev, const void* src, void* dst, size_t n, float alpha, float beta, uintptr_t stream);

/* ---- gather-reduce variant ------------------------------------------------------------------ */

/* Bytes of zero-initialised device workspace ktb_map_reduce_sum needs (per concurrent call). */
size_t ktb_reduce_workspace_bytes(void);
/* out[0] = sum_i op(src[i]).  Accumulator/out type: float for F32 and BF16 (per-thread fp32,
 * warp-shuffle tree, fp64 across CTAs — deterministic for a given n and device), int64 for
 * I32/I64 (exact, wrapping).  `out` may be a peer pointer (rank r writes root_out[r]).
 * `workspace` must be zero before first use; the kernel restores it to zero. */
int ktb_map_reduce_sum(int dev, int op, int dtype, const void* src, size_t n_elems,
                       double alpha, double beta, void* out, void* workspace, uintptr_t stream);
/* out[0] = sum of n partials (float or int64, per dtype rule above); the root-side final step. */
int ktb_reduce_partials(int dev, int dtype, const void* partials, int n, void* out, uintptr_t stream);

/* ---- pack / unpack: many tensors <-> one arena ------------------------------------------------- */

#define KTB_PACK_ALIGN 256
/* Computes offsets[i] (KTB_PACK_ALIGN-aligned, in order) for n segments; returns total bytes
 * needed in *total.  Pure host arithmetic (the layout half of pack). */
int ktb_pack_layout(const size_t* nbytes, int n, size_t* offsets, size_t* total);
/* arena[offsets[i] .. +nbytes[i]) = srcs[i][0..nbytes[i]) for all i, as one or more segmented
 * copy launches.  If `offsets` was not pre-filled pass compute_layout=1 to fill it here. */
int ktb_pack(int dev, const void* const* srcs, const size_t* nbytes, int n, void* arena,
             size_t arena_bytes, size_t* offsets, int compute_layout, uintptr_t stream);
int ktb_unpack(int dev, const void* arena, const size_t* offsets, const size_t* nbytes, int n,
               void* const* dsts, uintptr_t stream);
/* Batched map: n independent calls dst_i = op(src_i) (n_elems[i] elements each) in as few
 * launches as possible — the coalesced form of many small remote calls. */
int ktb_map_batch(int dev, int op, int dtype, const void* const* srcs, void* const* dsts,
                  const size_t* n_elems, int n, double alpha, double beta, uintptr_t stream);

/* ---- multi-GPU data movement over NVLink / NVSwitch ---------------------------------------------- */

/* SPMD broadcast (reference semantics: every rank sees the full args): one kernel on `root`
 * reads src once and peer-stores it into every dsts[k] (k < n_dst; entries equal to src are
 * skipped).  All dsts must be mapped on `root`. */
int ktb_broadcast(int root, const void* src, void* const* dsts, int n_dst, size_t nbytes,
                  uintptr_t stream);

/* Fused scatter → map → gather for a registered op, single controller process:
 * rank r (device devs[r]) pulls its torch.chunk shard of src_root straight out of the root
 * GPU's memory, applies op, and pushes the result into dst_root at the same offset.  No
 * staging copies: root HBM is read once and written once.  streams[r] is the stream on
 * devs[r], used verbatim (0 = legacy default stream); streams == NULL → library-owned streams.  The call is ordered after prior work on
 * streams[root_rank] and that stream is ordered after all ranks' work on return.
 * `granule` = elements per indivisible unit (a dim-0 row): shards are ktb_shard_bounds over
 * n_elems/granule units, i.e. exactly `x.chunk(world)` along dim 0; n_elems % granule must be 0. */
int ktb_scatter_map_gather(int op, int dtype, const void* src_root, void* dst_root, size_t n_elems,
                           size_t granule, double alpha, double beta, int n_ranks, const int* devs,
                           int root_rank, int variant, const uintptr_t* streams);
/* Gather-reduce variant: rank r reduces op(shard r) and writes partials_root[r]; the root then
 * reduces the n_ranks partials into out_root[0].  workspaces[r] as in ktb_map_reduce_sum. */
int ktb_scatter_map_reduce(int op, int dtype, const void* src_root, size_t n_elems, size_t granule,
                           double alpha, double beta, int n_ranks, const int* devs, int root_rank,
                           void* partials_root, void* out_root, void* const* workspaces,
                           const uintptr_t* streams);

/* ---- push/push pipeline: in-kernel flag synchronisation, no host sync on the data path ----------- */

/* Bytes of a control block (zero-initialised device memory; one per rank, one for the root). */
size_t ktb_push_control_bytes(void);
/* ROOT side of call number `seq` (1,2,3,... — every participant counts calls identically): for each
 * of n_chunks pieces, peer-store the piece of every non-root rank's shard into
 * stage_peer[r] + (seq&1)*stage_stride and publish ready[chunk] = seq in ctrl_peer[r].  The kernel
 * itself waits for ack[r] >= seq-2 (in ctrl_root) before overwriting a staging half.
 * stage_peer[r] / ctrl_peer[r] are pointers valid on root_dev (peer access or CUDA IPC). */
int ktb_push_scatter(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype,
                     int n_ranks, int root_rank, void* const* stage_peer, size_t stage_stride,
                     void* const* ctrl_peer, void* ctrl_root, int n_chunks, unsigned long long seq,
                     uintptr_t stream);
/* The same root side with pieces of EXACTLY chunk_elems elements per rank (n_chunks = ceil(largest shard /
 * chunk_elems) <= 64): for consumers that need whole work units per piece (ktb_mlp_bf16_pushed: GEMM row chunks).
 * ctas_per_sm caps the persistent grid (0 = library default) so the root's own compute keeps its share of every SM.
 * A rank whose stage_peer[r] is NULL is skipped (also in ktb_push_scatter / ktb_push_scatter_ce): two calls with
 * complementary NULL masks split the ranks between engines (hybrid copy-engine + SM scatter). */
int ktb_push_scatter_chunked(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype,
                             int n_ranks, int root_rank, void* const* stage_peer, size_t stage_stride,
                             void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems, int ctas_per_sm,
                             unsigned long long seq, uintptr_t stream);
/* Copy-engine form of the chunked root side: every piece is a cudaMemcpyPeerAsync on a per-destination library
 * stream of the root followed by a one-thread flag publish, issued chunk-major; NO SM of the root moves data, so its
 * own compute (rank 0's GEMMs in ktb_mlp_bf16_pushed deployments) keeps the whole GPU.  `stream` is ordered before
 * (sources ready) and after (sources reusable) the copies.  devs[r] = device of rank r. */
int ktb_push_scatter_ce(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype, int n_ranks,
                        int root_rank, const int* devs, void* const* stage_peer, size_t stage_stride,
                        void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems, unsigned long long seq,
                        uintptr_t stream);
/* RANK side: for each piece, spin in-kernel until ready[chunk] >= seq, then
 * dst_root_shard[piece] = op(stage_local[piece]) (peer stores into the root's result arena); after the
 * last piece publish ack[rank] = seq in the root's control block (ctrl_root_peer). */
int ktb_push_consume(int dev, int op, int dtype, const void* stage_local, size_t stage_stride,
                     void* dst_root_shard, size_t shard_elems, double alpha, double beta,
                     void* ctrl_local, void* ctrl_root_peer, int rank, int n_chunks,
                     unsigned long long seq, uintptr_t stream);
/* ROOT: stream-ordered completion of call `seq` (spins until every ack[r] >= seq). */
int ktb_push_wait(int root_dev, void* ctrl_root, int n_ranks, int root_rank, unsigned long long seq,
                  uintptr_t stream);
/* Synchronously read a control block's sticky status: 0 healthy, 1 = an in-kernel wait timed out. */
int ktb_push_status(int dev, const void* ctrl, unsigned int* out);

/* ---- host-resident args/results (the reference's client lives outside the GPU) -------------------- */

/* dst_host = op(src_host) with both buffers in pinned host memory, chunked through
 * device staging buffers (each >= 2*chunk_bytes) on three library streams so that H2D copy,
 * kernel and D2H copy of successive chunks overlap (PCIe is full duplex).  Synchronous:
 * returns when dst_host is complete. */
int ktb_map_host(int dev, int op, int dtype, const void* src_host, void* dst_host, size_t n_elems,
                 double alpha, double beta, size_t chunk_bytes, void* stage_in, void* stage_out);

/* The same for a sharded call on n_ranks DISTINCT devices: rank r's `x.chunk(n_ranks)[r]` (granule as in
 * ktb_scatter_map_gather) moves host → devs[r] → host over that GPU's own PCIe link, each pipeline enqueued by a
 * persistent library issue thread bound to the CPUs of that GPU's NUMA node (all links run concurrently).
 * stage_in[r] / stage_out[r] are device buffers of >= 2*chunk_bytes on devs[r].  Synchronous. */
int ktb_map_host_multi(int op, int dtype, const void* src_host, void* dst_host, size_t n_elems,
                       size_t granule, double alpha, double beta, int n_ranks, const int* devs,
                       size_t chunk_bytes, void* const* stage_in, void* const* stage_out);

/* ---- bf16 MLP policy (BASELINE config C4) ---------------------------------------------------------- */

/* logits[M,d_out] = W3·relu(W2·relu(W1·obs^T)) with bf16 storage, fp32 accumulation on wgmma
 * tensor cores (TMA-fed warp-specialised CTAs), activations rounded to bf16 between layers.
 * ktb_mlp_bf16, _staged and _pushed are the bias-free, 64-wide, logits-only case of the policy form
 * below (ktb_mlp_bf16_policy, _policy_pushed), run by the same kernel.
 * W_l is [d_l, d_{l-1}] row-major (nn.Linear layout).  This build: any M, d_in % 64 == 0,
 * d_hidden % 256 == 0 (KTB_ERR_ARG otherwise), d_out == 64 (KTB_ERR_UNSUPPORTED otherwise); every
 * pointer 16-byte aligned (KTB_ERR_ARG).  Rows are processed in chunks (16 896 rows by default), each
 * layer of a chunk as one GEMM launch over 128-row tiles; a tile is computed the same way whatever the
 * chunking, so every chunk size and every form below give bit-identical logits.  Each layer's result
 * is act(fp32 sum of the exact bf16 products) rounded to nearest-even bf16.  Writes stay inside
 * logits[M*d_out] and `scratch`, which holds 2*min(M, chunk)*d_hidden bf16 (ktb_mlp_scratch_bytes).
 * Replaces the user's nn.Sequential policy inside execute_callable_async
 * (kt/serving/http_server.py:1845-1891). */
size_t ktb_mlp_scratch_bytes(size_t M, int d_hidden);
int ktb_mlp_bf16(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                 const void* W1, const void* W2, const void* W3, void* logits, void* scratch,
                 uintptr_t stream);
/* Scatter-fused form for a rank whose observations live on the ROOT GPU: row chunks are pulled
 * peer → local into `stage` (ktb_mlp_stage_bytes, double-buffered; NULL is KTB_ERR_ARG) on a library
 * side stream while the previous chunk computes; `logits` may be a peer pointer (fused gather). */
size_t ktb_mlp_stage_bytes(size_t M, int d_in);
int ktb_mlp_bf16_staged(int dev, const void* obs_peer, size_t M, int d_in, int d_hidden, int d_out,
                        const void* W1, const void* W2, const void* W3, void* logits, void* scratch,
                        void* stage, uintptr_t stream);

/* Push-fed form for a rank whose observation rows are PUSHED by the root (ktb_push_scatter_chunked with
 * chunk_elems = chunk_rows * d_in into stage_local, double-buffered by call parity with stride stage_stride):
 * before each row chunk's GEMMs a one-warp kernel waits in-stream for ready[chunk] >= seq; the logits are stored
 * straight into `logits` (a peer pointer into the root's result: fused gather) and ack[rank] = seq is published in
 * the root's control block behind the last chunk.  Root NVLink egress carries posted writes only.
 * Requires M % 128 == 0 (a root routes other shards to the staged form), chunk_rows a positive multiple
 * of 128, ceil(M / chunk_rows) <= 64, M*d_in*2 <= stage_stride and stage_local, weights and scratch
 * 16-byte aligned (KTB_ERR_ARG otherwise); d_out == 64 (KTB_ERR_UNSUPPORTED otherwise).  `scratch`
 * holds 2*min(chunk_rows, M)*d_hidden bf16: it follows this call's chunk_rows, not the chunk of
 * ktb_mlp_scratch_bytes. */
int ktb_mlp_bf16_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden,
                        int d_out, const void* W1, const void* W2, const void* W3, void* logits, void* scratch,
                        void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq,
                        uintptr_t stream);

/* Policy form: the nn.Linear policy  Linear(d_in, d_hidden) → ReLU → Linear(d_hidden, d_hidden) → ReLU →
 * Linear(d_hidden, d_out)  with biases, a head of any width 1 <= d_out <= 256, and greedy actions.
 *   - Layer l is act(fp32 sum of the exact bf16 products + b_l) rounded ONCE to nearest-even bf16: the bias
 *     joins the fp32 accumulator before the ReLU (F.linear / nn.Linear, one rounding).  This differs from
 *     `x @ w.t() + b` written as two eager ops, which rounds twice.  ReLU is fmaxf, as in ktb_mlp_bf16.
 *   - b1 [d_hidden], b2 [d_hidden], b3 [d_out] bf16; each may be NULL (no bias on that layer).
 *   - logits [M, d_out] bf16 and/or actions [M] int64; either may be NULL, not both.  actions[i] =
 *     torch.argmax(logits[i]) over the ROUNDED logits: ties go to the lowest index, NaN is greater than any
 *     number (the first NaN wins), -0.0 == +0.0.  With logits NULL no logits are written anywhere.  Both may be
 *     peer pointers (fused gather).
 *   - d_out <= 0 is KTB_ERR_ARG, d_out > 256 KTB_ERR_UNSUPPORTED; d_in and d_hidden as ktb_mlp_bf16.
 *   - logits and the biases need 2-byte alignment (a rank's rows of a root result start at b*d_out*2 bytes),
 *     actions 8-byte; obs, weights, scratch and stage 16-byte (KTB_ERR_ARG).  scratch and stage are sized as
 *     for ktb_mlp_bf16 / _staged (ktb_mlp_scratch_bytes, ktb_mlp_stage_bytes).
 *   - stage == NULL is the plain form (obs local); otherwise the staged form of ktb_mlp_bf16_staged.
 *   - Writes stay inside logits[M*d_out], actions[M], scratch and stage.  Every chunking and form gives identical
 *     bits, and with no biases, d_out == 64 and logits only the logits equal ktb_mlp_bf16's bit for bit. */
int ktb_mlp_bf16_policy(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                        const void* W1, const void* b1, const void* W2, const void* b2,
                        const void* W3, const void* b3, void* logits, int64_t* actions,
                        void* scratch, void* stage, uintptr_t stream);
/* Push-fed policy form: ktb_mlp_bf16_pushed's contract (M % 128 == 0, chunk_rows, stage_stride, control blocks,
 * scratch of 2*min(chunk_rows, M)*d_hidden bf16) with the biases and outputs of ktb_mlp_bf16_policy.  An empty
 * shard (M == 0) may pass NULL outputs. */
int ktb_mlp_bf16_policy_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                               int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                               const void* b2, const void* W3, const void* b3, void* logits, int64_t* actions,
                               void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                               unsigned long long seq, uintptr_t stream);

/* Sampling form: the policy above with actions SAMPLED from softmax(logits) by Gumbel-max, and the log-probability
 * of each sampled action.  For the call's global row i (row_base + the row's index in this call) and head column j:
 *   - x = Philox4x32-10(counter = (i mod 2^32, i >> 32, j >> 1, 0), key = (seed mod 2^32, seed >> 32)), output word
 *     j & 1.  The round is Random123's (multipliers 0xD2511F53, 0xCD9E8D57; key increments 0x9E3779B9, 0xBB67AE85),
 *     the round of curand_philox4x32_x.h.
 *   - u = (2*(x >> 9) + 1) * 2^-24, exact in fp32 and strictly inside (0, 1); g = -log(-log(u)) in fp32 (logf, no
 *     fast-math), finite, within about [-2.81, 16.6].
 *   - actions[i] = argmax_j fp32(float(logit_j) + g_j) over j < d_out, where logit_j is the bf16-rounded head output
 *     (the value ktb_mlp_bf16_policy stores), under the torch.argmax rules of the greedy actions.
 *   - log_probs[i] = logit_a - m - log(sum_j exp(logit_j - m)) in fp32, m the row's largest logit: torch.log_softmax
 *     (logits.float(), -1)[a].  NaN on rows with a NaN or +inf logit and on rows whose logits are all -inf, as in
 *     torch; -inf logits (action masking through b3) are never sampled while the row has a finite logit.
 *   - The noise depends on (seed, i, j) only: every chunk size, form (plain, staged, pushed), rank count and device
 *     gives the same bits when each shard passes its first global row as row_base.  A new seed draws new samples.
 * No logits are written.  actions [M] int64 (8-byte aligned) and log_probs [M] fp32 (4-byte aligned) may be peer
 * pointers; either one NULL with M > 0 is KTB_ERR_ARG.  Every other argument is checked as in ktb_mlp_bf16_policy
 * (d_out > 256 is KTB_ERR_UNSUPPORTED).  Writes stay inside actions[M], log_probs[M], scratch and stage. */
int ktb_mlp_bf16_policy_sample(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                               const void* W1, const void* b1, const void* W2, const void* b2,
                               const void* W3, const void* b3, uint64_t seed, uint64_t row_base,
                               int64_t* actions, float* log_probs, void* scratch, void* stage, uintptr_t stream);
/* Push-fed sampling form: ktb_mlp_bf16_policy_pushed's arguments with (seed, row_base, actions, log_probs) in place
 * of (logits, actions).  An empty shard (M == 0) may pass NULL outputs. */
int ktb_mlp_bf16_policy_sample_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                      int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                      const void* b2, const void* W3, const void* b3, uint64_t seed,
                                      uint64_t row_base, int64_t* actions, float* log_probs, void* scratch,
                                      void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                      unsigned long long seq, uintptr_t stream);

/* Gaussian form: the policy above as the mean of a diagonal Gaussian with a state-independent log standard deviation
 * log_std [d_out] (fp32), as in PPO's continuous policies.  For the call's global row i (row_base + the row's index
 * in this call) and head column j:
 *   - x = Philox4x32-10(counter = (i mod 2^32, i >> 32, j >> 1, 1), key = (seed mod 2^32, seed >> 32)), output word
 *     j & 1: the Philox of the sampling form, with counter word 3 = 1, so that one seed never gives the Gaussian and
 *     the Gumbel heads the same uniforms.
 *   - u = (2*(x >> 9) + 1) * 2^-24, exact in fp32, strictly inside (0, 1) and never 0.5; z = normcdfinvf(u) in fp32
 *     (no fast-math), never 0 and within +-5.29471 (= Phi^-1(1 - 2^-24)): the tails beyond (probability mass about
 *     1.2e-7) are never drawn.
 *   - sigma_j = expf(log_std[j]); actions[i, j] = __fadd_rn(mu_ij, __fmul_rn(sigma_j, z_ij)) (no FMA contraction),
 *     where mu_ij is the bf16-rounded head output (the value ktb_mlp_bf16_policy stores).
 *   - log_probs[i] = -sum_j (0.5*z_ij^2 + log_std[j]) - d_out*0.5*log(2*pi) in fp32: Normal(mu, sigma).log_prob(a)
 *     .sum(-1), computed from z, so it does not depend on mu.
 *   - IEEE cases: log_std[j] = -inf gives sigma = 0, actions[i, j] == mu_ij as a value and log_probs = +inf;
 *     log_std[j] = +inf gives +-inf actions (z != 0) and log_probs = -inf; a NaN log_std[j] gives a NaN column and
 *     NaN log-probabilities.  A NaN or +-inf logit affects its own action only; the row's log-probability is unchanged.
 *   - The noise depends on (seed, i, j) only: every chunk size, form (plain, staged, pushed), rank count and device
 *     gives the same bits when each shard passes its first global row as row_base.
 * No logits are written.  actions [M, d_out] fp32 (4-byte aligned; may be a peer pointer), log_probs [M] fp32 (4-byte
 * aligned) and log_std [d_out] fp32 (4-byte aligned): any one NULL with M > 0 is KTB_ERR_ARG.  Every other argument is
 * checked as in ktb_mlp_bf16_policy (d_out > 256 is KTB_ERR_UNSUPPORTED).  Writes stay inside actions[M, d_out],
 * log_probs[M], scratch and stage. */
int ktb_mlp_bf16_policy_gaussian(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                 const void* W1, const void* b1, const void* W2, const void* b2,
                                 const void* W3, const void* b3, const float* log_std, uint64_t seed,
                                 uint64_t row_base, float* actions, float* log_probs, void* scratch, void* stage,
                                 uintptr_t stream);
/* Push-fed Gaussian form: ktb_mlp_bf16_policy_sample_pushed's arguments with log_std before the seed and fp32
 * actions [M, d_out].  An empty shard (M == 0) may pass NULL outputs. */
int ktb_mlp_bf16_policy_gaussian_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                        int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                        const void* b2, const void* W3, const void* b3, const float* log_std,
                                        uint64_t seed, uint64_t row_base, float* actions, float* log_probs,
                                        void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                        size_t chunk_rows, unsigned long long seq, uintptr_t stream);

#ifdef __cplusplus
}
#endif
#endif /* KTB200_H */
