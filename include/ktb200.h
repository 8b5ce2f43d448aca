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
 * (float for F32/BF16/F16, int64 for I32/I64).  For I32/I64 they must hold integers: the kernels take
 * (long long)alpha and compute modulo 2^32 / 2^64, so pass the scalar reduced to that width's signed range,
 * where it is exact in a double for I32 and, for I64, exact only when |value| <= 2^53 or otherwise representable.
 * KTB_U8 supports KTB_OP_IDENTITY only.
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
/* ktb_push_scatter_ce with a second source per row for the masked MLP heads: row i of obs (granule elements) has
 * row_bytes bytes at mask_root + i*row_bytes (the legal-action mask, row_bytes = d_out).  On each rank's copy-engine
 * stream, after the same wait for ack[r] >= seq-2, chunk c's mask rows are copied to stage_peer[r] + (seq&1)*stage_stride
 * + mask_offset + (the chunk's first row in the shard)*row_bytes, and ready[c] is published behind both copies.  After
 * every check of ktb_push_scatter_ce, in its order: a NULL mask_root with n_elems > 0, row_bytes == 0, chunk_elems not
 * a multiple of granule, and for a served rank mask_offset < its shard's bytes or mask_offset + rows*row_bytes >
 * stage_stride are KTB_ERR_ARG. */
int ktb_push_scatter_ce_masked(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype,
                               int n_ranks, int root_rank, const int* devs, void* const* stage_peer,
                               size_t stage_stride, void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems,
                               const void* mask_root, size_t row_bytes, size_t mask_offset, unsigned long long seq,
                               uintptr_t stream);
/* ktb_push_scatter_ce with n_sides (1 or 2) per-row side sources, the side inputs of the push-fed MLP heads
 * (ktb_mlp_bf16_pushed): row i of obs has side_row_bytes[k] bytes at side_src[k] +
 * i*side_row_bytes[k], copied chunk by chunk, after the same wait for ack[r] >= seq-2, to stage_peer[r] +
 * (seq&1)*stage_stride + side_offset[k] + (the chunk's first row in the shard)*side_row_bytes[k]; ready[c] is
 * published behind every copy of chunk c.  ktb_push_scatter_ce_masked is its one-side case.  After every check of
 * ktb_push_scatter_ce, in its order: n_sides outside [1, 2] or a NULL array; then per side in order a NULL source with
 * n_elems > 0, side_row_bytes == 0 or chunk_elems not a multiple of granule; then for each served rank a side that
 * overlaps its shard's rows, ends past stage_stride, or overlaps an earlier side, are KTB_ERR_ARG. */
int ktb_push_scatter_ce_sides(int root_dev, const void* src_root, size_t n_elems, size_t granule, int dtype,
                              int n_ranks, int root_rank, const int* devs, void* const* stage_peer, size_t stage_stride,
                              void* const* ctrl_peer, void* ctrl_root, size_t chunk_elems, int n_sides,
                              const void* const* side_src, const size_t* side_row_bytes, const size_t* side_offset,
                              unsigned long long seq, uintptr_t stream);
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

/* dst_host = op(src_host) with both buffers in pinned host memory, sharded over n_ranks: rank r's
 * `x.chunk(n_ranks)[r]` (granule as in ktb_scatter_map_gather) moves host → devs[r] → host over that GPU's own
 * PCIe link, chunked through device staging buffers stage_in[r] / stage_out[r] (each >= 2*chunk_bytes, on
 * devs[r]) on three library streams so that H2D copy, kernel and D2H copy of successive chunks overlap (PCIe is
 * full duplex).  Each device's pipeline is enqueued by a persistent library issue thread bound to the CPUs of
 * that GPU's NUMA node (all links run concurrently); the first device's runs on the calling thread.  A one-GPU
 * call is n_ranks = 1, devs = {dev}, granule = 1.  Synchronous: returns when dst_host is complete.
 *   - Rank subsets: a rank whose stage_in[r] and stage_out[r] are both NULL is not part of the call and its shard of
 *     dst_host is left alone; exactly one of the two NULL is KTB_ERR_ARG; every rank NULL moves nothing (KTB_OK).
 *   - devs may repeat: the selected ranks of one device run one after another in rank order (they share its
 *     streams, events and staging, so they may share staging buffers too). */
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
 * of 128, ceil(M / chunk_rows) <= 64, M*d_in*2 <= stage_stride, stage_stride % 16 == 0 (each call's half is
 * 16-byte aligned) and stage_local, weights and scratch 16-byte aligned (KTB_ERR_ARG otherwise, before anything
 * is enqueued); d_out == 64 (KTB_ERR_UNSUPPORTED otherwise).  `scratch`
 * holds 2*min(chunk_rows, M)*d_hidden bf16: it follows this call's chunk_rows, not the chunk of
 * ktb_mlp_scratch_bytes.
 * Side inputs of the push-fed heads: a head's per-row inputs (its sides, up to two, named by each family below) are
 * pushed beside the rows into the same staging half (ktb_push_scatter_ce_sides puts them there), and the rank reads
 * them at stage_local + (seq & 1)*stage_stride + the side's offset argument, never from a peer.  Each side holds M rows
 * of its bytes per row and needs its alignment; a side that starts inside the rows (offset < M*d_in*2), ends past
 * stage_stride, starts at an offset that is not a multiple of its alignment, or overlaps an earlier side is
 * KTB_ERR_ARG.  These checks come right after those of stage_stride, before every check of the head's own arguments, so
 * a call with a bad side and another defect (say an unsupported d_out) may report the side's KTB_ERR_ARG first. */
int ktb_mlp_bf16_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden,
                        int d_out, const void* W1, const void* W2, const void* W3, void* logits, void* scratch,
                        void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq,
                        uintptr_t stream);

/* Policy form: the nn.Linear policy  Linear(d_in, d_hidden) → ReLU → Linear(d_hidden, d_hidden) → ReLU →
 * Linear(d_hidden, d_out)  with biases, a head of any width 1 <= d_out <= 256, and greedy actions.
 *   - Layer l is act(fp32 sum of the exact bf16 products + b_l) rounded ONCE to nearest-even bf16: the bias
 *     joins the fp32 accumulator before the ReLU (F.linear / nn.Linear, one rounding).  This differs from
 *     `x @ w.t() + b` written as two eager ops, which rounds twice.  ReLU is torch.relu, as in ktb_mlp_bf16: a NaN
 *     pre-activation stays NaN (max.NaN, not fmaxf), +inf stays +inf, -inf becomes 0.
 *   - IEEE special values follow torch (measured on H100 80GB HBM3): the tensor cores keep NaN and +-inf from their
 *     bf16 inputs and give NaN for inf * 0 and +inf - inf; an fp32 sum past FLT_MAX is +-inf; a result on the bf16
 *     overflow tie rounds to +-inf; subnormal inputs and results are not flushed.  So a NaN observation row gives NaN
 *     outputs in that row only, and a NaN weight or bias of any layer gives NaN outputs in every row it reaches.
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
 *     torch; -inf logits (one mask for every row through b3; per-row masks: the _masked forms below) are never
 *     sampled while the row has a finite logit.
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

/* Masked forms: ktb_mlp_bf16_policy and ktb_mlp_bf16_policy_sample with a per-row legal-action mask.
 *   - mask [M, d_out] bytes, row-major (torch.bool): any nonzero byte means legal.  It may be a peer pointer (the
 *     rank's rows of the root's mask); it is read once per row, only at rows < M and columns < d_out.
 *   - The head computes exactly y.masked_fill(~legal, -inf) on its bf16-rounded output y (the value
 *     ktb_mlp_bf16_policy stores), and every rule of the unmasked entry then applies to those masked logits: logits
 *     hold bf16 -inf in illegal columns; actions are torch.argmax of the masked logits; the sampling form draws
 *     Gumbel-max over them with the same Philox counters, and log_probs = log_softmax(masked.float())[a].
 *   - A row with no legal action gets action 0 (and a NaN log-probability when sampled); a row with exactly one legal
 *     action, whose logit is finite, gets that action with log-probability exactly 0.0.  A NaN or +inf logit in an
 *     illegal column has no effect.  An all-legal mask gives the bits of the unmasked entry.
 *   - A NULL mask with M > 0 is KTB_ERR_ARG, checked after every check of the unmasked entry, in the same order. */
int ktb_mlp_bf16_policy_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                               const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                               const void* b3, const uint8_t* mask, void* logits, int64_t* actions, void* scratch,
                               void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                      const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                      const void* b3, const uint8_t* mask, uint64_t seed, uint64_t row_base,
                                      int64_t* actions, float* log_probs, void* scratch, void* stage,
                                      uintptr_t stream);
/* Push-fed masked forms: the _pushed entries' arguments with mask_offset after b3, the offset of their one side
 * (ktb_mlp_bf16_pushed): the mask, d_out bytes per row, any alignment. */
int ktb_mlp_bf16_policy_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                      int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                      const void* b2, const void* W3, const void* b3, size_t mask_offset, void* logits,
                                      int64_t* actions, void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                      size_t chunk_rows, unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                             int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                             const void* b2, const void* W3, const void* b3, size_t mask_offset,
                                             uint64_t seed, uint64_t row_base, int64_t* actions, float* log_probs,
                                             void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                             size_t chunk_rows, unsigned long long seq, uintptr_t stream);

/* Value forms: the sampling, masked sampling and Gaussian entries with a value head V(s) on the same trunk, the critic
 * nn.Linear(d_hidden, 1) of a shared-trunk actor-critic.
 *   - W3v [d_out + 1, d_hidden] bf16 is the policy's W3 with the critic's weight wv [1, d_hidden] stacked under it, and
 *     b3v [d_out + 1] is b3 with the critic's bias bv after it, or NULL when neither has a bias.  d_out stays the
 *     policy's width.
 *   - values[i] = fp32(bf16(h2_i . wv + bv)): column d_out of the head, rounded once to bf16 with the bias in the fp32
 *     accumulator (F.linear), then widened exactly to fp32.  It is the value column d_out of ktb_mlp_bf16_policy's
 *     logits for the same W3v and b3v.
 *   - Actions and log-probabilities have the bits of the entry without a value head over W3 and b3: the value column
 *     is never ranked, sampled, summed into the softmax or given a log_std, and it draws no Philox noise.  A
 *     legal-action mask [M, d_out] never touches the values.
 *   - values [M] fp32 follows log_probs and may be a peer pointer.  With M > 0, a NULL or not 4-byte aligned values is
 *     KTB_ERR_ARG and d_out = 256 is KTB_ERR_UNSUPPORTED (the d_out + 1 columns must fit one 256-wide tile); these are
 *     checked after every check of the entry without a value head.  An empty pushed shard (M == 0) may pass NULL
 *     outputs and still publishes its ack.  Writes stay inside the outputs of that entry, values[M], scratch and
 *     stage. */
int ktb_mlp_bf16_policy_sample_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                     const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v,
                                     const void* b3v, uint64_t seed, uint64_t row_base, int64_t* actions,
                                     float* log_probs, float* values, void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                            int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                            const void* b2, const void* W3v, const void* b3v, uint64_t seed,
                                            uint64_t row_base, int64_t* actions, float* log_probs, float* values,
                                            void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                            size_t chunk_rows, unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_masked_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                            const void* W1, const void* b1, const void* W2, const void* b2,
                                            const void* W3v, const void* b3v, const uint8_t* mask, uint64_t seed,
                                            uint64_t row_base, int64_t* actions, float* log_probs, float* values,
                                            void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_masked_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                   int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                   const void* W2, const void* b2, const void* W3v, const void* b3v,
                                                   size_t mask_offset, uint64_t seed, uint64_t row_base,
                                                   int64_t* actions, float* log_probs, float* values, void* scratch,
                                                   void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                   unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v,
                                       const void* b3v, const float* log_std, uint64_t seed, uint64_t row_base,
                                       float* actions, float* log_probs, float* values, void* scratch, void* stage,
                                       uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                              int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                              const void* b2, const void* W3v, const void* b3v, const float* log_std,
                                              uint64_t seed, uint64_t row_base, float* actions, float* log_probs,
                                              float* values, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                              int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream);

/* State-dependent Gaussian forms: the Gaussian entries with a per-row log standard deviation from a second linear head
 * on the same trunk, clamped, and optionally tanh-squashed actions (SAC's actor).  Each takes the arguments of its
 * _gaussian counterpart with W3s / b3s (W3sv / b3sv) in place of W3 / b3 (W3v / b3v) and (log_std_min, log_std_max,
 * squash) in place of log_std.  d_out stays the action width.
 *   - W3s [2*d_out, d_hidden] bf16 interleaves the mean's and the log-std's weights: row 2j is w3[j], row 2j + 1 is
 *     w_ls[j]; b3s [2*d_out] likewise interleaves b3 and b_ls, or is NULL when neither has a bias.  With a value head,
 *     W3sv / b3sv have the critic's row 2*d_out after them, and values are as in the value forms.
 *   - mu_ij and l_ij are the bf16-rounded head outputs of rows 2j and 2j + 1 (ktb_mlp_bf16_policy's logits over W3s);
 *     lc = l clamped to [log_std_min, log_std_max] by comparisons, so a NaN l stays NaN; infinite bounds clamp nothing.
 *   - z_ij is the noise of the Gaussian form for action column j (Philox word j & 1 of counter (i, j >> 1, 1)), and
 *     u = __fadd_rn(mu_ij, __fmul_rn(expf(lc), z_ij)), the Gaussian form's rounding.  actions[i, j] = tanhf(u) when
 *     squash != 0, u otherwise.  Squashed actions may be exactly +-1.0 in fp32.
 *   - log_probs[i] = -sum_j (0.5*z^2 + lc) - d_out*0.5*log(2*pi), and with squash also -sum_j c(u) with
 *     c(u) = 2*(log 2 - |u| - log1pf(expf(-2|u|))) = log(1 - tanh(u)^2) exactly (not SB3's log(1 - tanh^2 + 1e-6),
 *     which differs where 1 - tanh^2 nears 1e-6, |u| > about 7).  It is computed from u, so it stays finite where the
 *     action rounds to +-1.0.  Terms are summed per thread and then across 4 lanes, so the order differs from the
 *     Gaussian form's.
 *   - IEEE cases: a NaN l gives a NaN action in its column and a NaN log-probability.  An infinite log_std_max lets
 *     expf(lc) overflow to +inf: then u = +-inf, the action is +-1.0 (squashed) or +-inf, and c(u) = -inf makes
 *     the squashed log-probability +inf (NaN when lc is itself +inf: -inf + inf); unsquashed it is -inf only when lc
 *     is +inf.  lc = -inf gives sigma = 0, u == mu and an unsquashed log-probability of +inf.
 *   - With w_ls = 0 and b_ls = c, the unsquashed actions are those of the Gaussian form with log_std = c, bit for bit.
 *   - Checks: every check of the _gaussian counterpart first (log_std excepted), then, with M > 0: 2*d_out (+1 with
 *     a value head) > 256, that is d_out > 128 (> 127), is KTB_ERR_UNSUPPORTED; a NaN bound or log_std_min >
 *     log_std_max is KTB_ERR_ARG.  An empty pushed shard (M == 0) may pass NULL outputs and still publishes its ack.
 *     Writes stay inside actions[M, d_out], log_probs[M], values[M] (value forms), scratch and stage. */
int ktb_mlp_bf16_policy_gaussian_state(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3s,
                                       const void* b3s, float log_std_min, float log_std_max, int squash,
                                       uint64_t seed, uint64_t row_base, float* actions, float* log_probs,
                                       void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_state_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                              int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                              const void* b2, const void* W3s, const void* b3s, float log_std_min,
                                              float log_std_max, int squash, uint64_t seed, uint64_t row_base,
                                              float* actions, float* log_probs, void* scratch, void* ctrl_local,
                                              void* ctrl_root_peer, int rank, size_t chunk_rows,
                                              unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_state_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                             const void* W1, const void* b1, const void* W2, const void* b2,
                                             const void* W3sv, const void* b3sv, float log_std_min, float log_std_max,
                                             int squash, uint64_t seed, uint64_t row_base, float* actions,
                                             float* log_probs, float* values, void* scratch, void* stage,
                                             uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_state_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                    int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                    const void* W2, const void* b2, const void* W3sv,
                                                    const void* b3sv, float log_std_min, float log_std_max, int squash,
                                                    uint64_t seed, uint64_t row_base, float* actions,
                                                    float* log_probs, float* values, void* scratch, void* ctrl_local,
                                                    void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                    unsigned long long seq, uintptr_t stream);

/* Multi-discrete forms: the greedy and sampling entries above (masked, pushed and with a value head as they come) for
 * a MultiDiscrete(nvec) action space, one categorical sub-action per group of head columns.  Each takes the
 * arguments of its categorical counterpart with (nvec, n_groups) inserted after b3 (or b3v).
 *   - nvec [n_groups] int32 is a host array, read before the call returns.  Group g is the columns [lo_g, lo_g + n_g)
 *     with lo_g = n_0 + ... + n_{g-1}; the groups tile the policy's d_out columns (a value column lies outside them).
 *   - actions [M, n_groups] int64 (8-byte aligned; may be a peer pointer) holds group-relative actions in [0, n_g):
 *     the counterpart's rule applied to each group's columns alone.  Greedy: torch.argmax of the group's (masked)
 *     logits.  Sampled: Gumbel-max over the group's columns with the counterpart's noise (column j of global row i
 *     draws Philox word j & 1 of counter (i, j >> 1, 0)), each pair of columns drawn once.
 *   - log_probs [M] fp32: the sum, in fp32 and in group order starting from group 0's term, of each group's
 *     log_softmax(group.float())[a_g].  A group whose ranked values are all -inf (no legal column, or only -inf
 *     logits) takes action 0 and makes the row's log-probability NaN, as torch does.
 *   - logits (greedy entries only, may be NULL) are those of ktb_mlp_bf16_policy or its _masked form, bit for bit; a
 *     greedy entry needs logits or actions, as ktb_mlp_bf16_policy does.  values as in the value forms.
 *   - nvec = {d_out} gives the bits of the counterpart's outputs, and group g of any nvec gives, bit for bit, the
 *     action (minus lo_g) and log-probability of the counterpart under the mask legal & (column in group g).
 *   - Checks: every check of the counterpart first, then, with M > 0: a NULL nvec, n_groups outside [1, d_out], any
 *     nvec[g] < 1 or a sum other than d_out is KTB_ERR_ARG.  An empty pushed shard (M == 0) may pass NULL outputs and
 *     a NULL nvec and still publishes its ack.  Writes stay inside the counterpart's outputs with actions [M, n_groups],
 *     scratch and stage. */
int ktb_mlp_bf16_policy_multidiscrete(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                      const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                      const void* b3, const int32_t* nvec, int n_groups, void* logits,
                                      int64_t* actions, void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_multidiscrete_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                             int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                             const void* b2, const void* W3, const void* b3, const int32_t* nvec,
                                             int n_groups, void* logits, int64_t* actions, void* scratch,
                                             void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                             unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_multidiscrete_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                             const void* W1, const void* b1, const void* W2, const void* b2,
                                             const void* W3, const void* b3, const int32_t* nvec, int n_groups,
                                             const uint8_t* mask, void* logits, int64_t* actions, void* scratch,
                                             void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_multidiscrete_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                    int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                    const void* W2, const void* b2, const void* W3, const void* b3,
                                                    const int32_t* nvec, int n_groups, size_t mask_offset,
                                                    void* logits, int64_t* actions, void* scratch, void* ctrl_local,
                                                    void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                    unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                             const void* W1, const void* b1, const void* W2, const void* b2,
                                             const void* W3, const void* b3, const int32_t* nvec, int n_groups,
                                             uint64_t seed, uint64_t row_base, int64_t* actions, float* log_probs,
                                             void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                    int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                    const void* W2, const void* b2, const void* W3, const void* b3,
                                                    const int32_t* nvec, int n_groups, uint64_t seed,
                                                    uint64_t row_base, int64_t* actions, float* log_probs,
                                                    void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                                    size_t chunk_rows, unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden,
                                                    int d_out, const void* W1, const void* b1, const void* W2,
                                                    const void* b2, const void* W3, const void* b3,
                                                    const int32_t* nvec, int n_groups, const uint8_t* mask,
                                                    uint64_t seed, uint64_t row_base, int64_t* actions,
                                                    float* log_probs, void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete_masked_pushed(int dev, const void* stage_local, size_t stage_stride,
                                                           size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                                           const void* b1, const void* W2, const void* b2,
                                                           const void* W3, const void* b3, const int32_t* nvec,
                                                           int n_groups, size_t mask_offset, uint64_t seed,
                                                           uint64_t row_base, int64_t* actions, float* log_probs,
                                                           void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                                           int rank, size_t chunk_rows, unsigned long long seq,
                                                           uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete_value(int dev, const void* obs, size_t M, int d_in, int d_hidden,
                                                   int d_out, const void* W1, const void* b1, const void* W2,
                                                   const void* b2, const void* W3v, const void* b3v,
                                                   const int32_t* nvec, int n_groups, uint64_t seed,
                                                   uint64_t row_base, int64_t* actions, float* log_probs,
                                                   float* values, void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete_value_pushed(int dev, const void* stage_local, size_t stage_stride,
                                                          size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                                          const void* b1, const void* W2, const void* b2,
                                                          const void* W3v, const void* b3v, const int32_t* nvec,
                                                          int n_groups, uint64_t seed, uint64_t row_base,
                                                          int64_t* actions, float* log_probs, float* values,
                                                          void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                                          int rank, size_t chunk_rows, unsigned long long seq,
                                                          uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete_masked_value(int dev, const void* obs, size_t M, int d_in, int d_hidden,
                                                          int d_out, const void* W1, const void* b1, const void* W2,
                                                          const void* b2, const void* W3v, const void* b3v,
                                                          const int32_t* nvec, int n_groups, const uint8_t* mask,
                                                          uint64_t seed, uint64_t row_base, int64_t* actions,
                                                          float* log_probs, float* values, void* scratch, void* stage,
                                                          uintptr_t stream);
int ktb_mlp_bf16_policy_sample_multidiscrete_masked_value_pushed(
    int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_out,
    const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v, const void* b3v,
    const int32_t* nvec, int n_groups, size_t mask_offset, uint64_t seed, uint64_t row_base, int64_t* actions,
    float* log_probs, float* values, void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
    size_t chunk_rows, unsigned long long seq, uintptr_t stream);

/* Epsilon-greedy forms: the actor of a Q-network (DQN, Ape-X, R2D2), whose head outputs one Q-value per action.  Each
 * takes ktb_mlp_bf16_policy's arguments up to b3, then (masked forms) the legal-action mask, then
 * (const float* epsilon, uint64_t seed, uint64_t row_base, int64_t* actions, float* q, float* q_max), then scratch,
 * stage (NULL: the plain form) and stream.  For the call's global row i (row_base + the row's index in this call), head
 * column j < d_out and key = (seed mod 2^32, seed >> 32):
 *   - q_ij is the bf16-rounded head output (ktb_mlp_bf16_policy's logits); masked: q.masked_fill(~legal, -inf) as the
 *     _masked entries compute it.
 *   - The greedy action g_i is torch.argmax(q_i): ties to the lowest column, the first NaN wins, -0.0 == +0.0, and a
 *     row whose ranked values are all -inf, or that has no legal column, gets 0.
 *   - The coin: x = word 0 of Philox4x32-10((i mod 2^32, i >> 32, 0, 3), key), u_i = (2*(x >> 9) + 1)*2^-24; row i
 *     explores iff u_i < epsilon[i] as an fp32 compare, so epsilon <= 0 and a NaN epsilon never explore, epsilon >= 1
 *     always does, and P(explore) is the count of the 2^23 grid points below epsilon over 2^23.
 *   - The exploratory action e_i: w_ij = word j & 1 of counter (i mod 2^32, i >> 32, j >> 1, 2) as a uint32; e_i is
 *     the legal column with the largest w_ij, ties to the lowest column, 0 when the row has no legal column.  It is
 *     uniform over the legal columns (ties have probability below d^2*2^-33) and reads no Q-value, so NaN or +-inf
 *     Q-values do not change it.  Counter word 3 = 2 (exploration) and 3 (coin) never reuse the Gumbel (0) or
 *     Gaussian (1) uniforms of the same seed.  Only an exploring row draws words: one Philox call per column pair.
 *   - actions[i] = explore ? e_i : g_i (int64); q[i] = fp32(q_i[actions[i]]), the masked Q-value of the action taken
 *     widened exactly (-inf for column 0 of a row with no legal column); q_max[i] = fp32(q_i[g_i]), NaN when a legal
 *     column holds a NaN.  No logits are written: 16 B per row.
 *   - The draws depend on (seed, i, j) only: every chunk size, form, rank count and row_base split gives the same bits.
 *   - epsilon, actions, q and q_max may be peer pointers in the plain and staged forms.
 *   - Checks: every check of the greedy counterpart (ktb_mlp_bf16_policy or _masked) first, in its order (d_out > 256
 *     is KTB_ERR_UNSUPPORTED), then, with M > 0: a NULL or misaligned (4 bytes; actions 8) epsilon, actions, q or q_max
 *     is KTB_ERR_ARG.  Writes stay inside actions[M], q[M], q_max[M], scratch and stage. */
int ktb_mlp_bf16_policy_epsilon_greedy(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                       const void* b3, const float* epsilon, uint64_t seed, uint64_t row_base,
                                       int64_t* actions, float* q, float* q_max, void* scratch, void* stage,
                                       uintptr_t stream);
int ktb_mlp_bf16_policy_epsilon_greedy_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                              const void* W1, const void* b1, const void* W2, const void* b2,
                                              const void* W3, const void* b3, const uint8_t* mask,
                                              const float* epsilon, uint64_t seed, uint64_t row_base,
                                              int64_t* actions, float* q, float* q_max, void* scratch, void* stage,
                                              uintptr_t stream);
/* Push-fed epsilon-greedy forms: the _pushed entries' arguments with (mask_offset,) epsilon_offset after b3 in place of
 * the pointers, the offsets of their sides (ktb_mlp_bf16_pushed): the mask (masked form; d_out bytes per row, any
 * alignment), then epsilon (fp32, 4 bytes per row, 4-byte aligned).  An empty shard (M == 0) may pass NULL outputs and
 * still publishes its ack. */
int ktb_mlp_bf16_policy_epsilon_greedy_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                              int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                              const void* b2, const void* W3, const void* b3, size_t epsilon_offset,
                                              uint64_t seed, uint64_t row_base, int64_t* actions, float* q,
                                              float* q_max, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                              int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_epsilon_greedy_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                     int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                     const void* W2, const void* b2, const void* W3, const void* b3,
                                                     size_t mask_offset, size_t epsilon_offset, uint64_t seed,
                                                     uint64_t row_base, int64_t* actions, float* q, float* q_max,
                                                     void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                                     size_t chunk_rows, unsigned long long seq, uintptr_t stream);

/* Evaluating forms: the log-probability and the entropy of actions the caller already holds, under the categorical
 * (single or multi-discrete, masked or not) or the state-independent Gaussian policy, with no noise drawn and no logits
 * written: SB3's policy.evaluate_actions and RLlib's dist.logp / dist.entropy, forward only.
 * Categorical (ktb_mlp_bf16_policy_evaluate and its _masked, _value and _masked_value forms): ktb_mlp_bf16_policy's
 * arguments up to b3 (W3v / b3v in the value forms), then (const int32_t* nvec, int n_groups, [const uint8_t* mask,]
 * const int64_t* taken, float* log_probs, float* entropy, [float* values,] void* scratch, void* stage, uintptr_t stream).
 *   - y is the bf16-rounded head output (ktb_mlp_bf16_policy's logits); masked: y.masked_fill(~legal, -inf).
 *   - Groups as in the multi-discrete forms; nvec == NULL with n_groups == 0 is one group of the d_out columns.  taken
 *     [M] (no nvec) or [M, n_groups] int64 holds group-relative actions a_g.
 *   - For group g over columns [lo, hi) and its legal columns: m = their max (NaN skipped), S = sum (y == m ? 1 :
 *     expf(y - m)), T = sum w*(y - m) with w the term of S (one fused multiply-add; a -inf column adds 0 to both), in
 *     the sampling forms' per-thread and quad order.  Then, in this order of precedence: a_g outside [0, hi - lo) gives
 *     lp_g = H_g = NaN; no legal column, or m == -inf, gives lp_g = H_g = NaN (torch's log_softmax of an all -inf row);
 *     an illegal column lo + a_g gives lp_g = -inf; otherwise lp_g = y[lo + a_g] - m - logf(S), the expression of the
 *     sampling forms; and H_g = logf(S) - T / S.
 *   - log_probs[i] and entropy[i] are the fp32 sums over groups in group order, starting from group 0's term.  With a
 *     value head values[i] is computed as in the value forms.
 *   - So evaluating the actions a sampling form drew (same weights, mask and nvec) returns its log_probs bit for bit,
 *     NaN in the same rows.  A row with one legal column gives lp = 0 and H = 0 for that column; n equal logits give
 *     H = logf(n).  A NaN legal logit makes S, T, the row's lp (but an illegal action's -inf) and H NaN; a +inf logit
 *     makes T, H and the lp of a +inf column NaN, and the lp of a finite column -inf.
 *   - An action out of range is a caller error: it is not checked (that would need a host synchronisation) and gives a
 *     NaN row.
 * Gaussian (ktb_mlp_bf16_policy_gaussian_evaluate and its _value form): ktb_mlp_bf16_policy_gaussian's arguments up to
 * log_std, then (const float* taken, float* log_probs, float* entropy, [float* values,] void* scratch, void* stage,
 * uintptr_t stream).  There is no seed and no row_base.
 *   - mu is the bf16-rounded head output; taken [M, d_out] fp32.  z_j = __fdiv_rn(__fsub_rn(a_j, mu_j),
 *     expf(log_std[j])), with no FMA contraction.
 *   - log_probs[i] = -sum_j (0.5*z_j^2 + log_std[j]) - d_out*0.5*log(2*pi), in the Gaussian form's per-thread and quad
 *     order: Normal(mu, exp(log_std)).log_prob(taken).sum(-1).
 *   - entropy[i] = sum_j (log_std[j] + 0.5) + d_out*0.5*log(2*pi), the same value in every row: Normal.entropy().sum(-1).
 *   - IEEE cases follow the formulas: log_std[j] = -inf gives sigma = 0, z = +-inf (NaN where a_j == mu_j) and an
 *     lp of -inf (or NaN); a NaN log_std, action or mean makes lp NaN; H is NaN for a NaN log_std.
 * Checks: every check of the counterpart without evaluation first, in its order (ktb_mlp_bf16_policy or _masked; the
 * value forms' values and d_out = 256 KTB_ERR_UNSUPPORTED; ktb_mlp_bf16_policy_gaussian's log_std), then the nvec checks
 * of the multi-discrete forms unless nvec == NULL and n_groups == 0, then, with M > 0, a NULL or misaligned taken (8
 * bytes categorical, 4 Gaussian), log_probs or entropy (4 bytes) is KTB_ERR_ARG.  Every chunk size, form and row split
 * gives the same bits.  taken and the outputs may be peer pointers in the plain and staged forms.  Writes stay inside
 * log_probs[M], entropy[M], values[M] (value forms), scratch and stage. */
int ktb_mlp_bf16_policy_evaluate(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                                 const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                                 const int32_t* nvec, int n_groups, const int64_t* taken, float* log_probs,
                                 float* entropy, void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_evaluate_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                        const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                        const void* b3, const int32_t* nvec, int n_groups, const uint8_t* mask,
                                        const int64_t* taken, float* log_probs, float* entropy, void* scratch,
                                        void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_evaluate_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                       const void* W1, const void* b1, const void* W2, const void* b2, const void* W3v,
                                       const void* b3v, const int32_t* nvec, int n_groups, const int64_t* taken,
                                       float* log_probs, float* entropy, float* values, void* scratch, void* stage,
                                       uintptr_t stream);
int ktb_mlp_bf16_policy_evaluate_masked_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                              const void* W1, const void* b1, const void* W2, const void* b2,
                                              const void* W3v, const void* b3v, const int32_t* nvec, int n_groups,
                                              const uint8_t* mask, const int64_t* taken, float* log_probs,
                                              float* entropy, float* values, void* scratch, void* stage,
                                              uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_evaluate(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                          const void* W1, const void* b1, const void* W2, const void* b2,
                                          const void* W3, const void* b3, const float* log_std, const float* taken,
                                          float* log_probs, float* entropy, void* scratch, void* stage,
                                          uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_evaluate_value(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                                const void* W1, const void* b1, const void* W2, const void* b2,
                                                const void* W3v, const void* b3v, const float* log_std,
                                                const float* taken, float* log_probs, float* entropy, float* values,
                                                void* scratch, void* stage, uintptr_t stream);
/* Push-fed evaluating forms: the _pushed entries' arguments with the evaluating arguments above after b3 (b3v), and
 * (mask_offset,) taken_offset in place of the pointers, the offsets of their sides (ktb_mlp_bf16_pushed): the mask
 * (masked forms; d_out bytes per row, any alignment), then taken (8*max(n_groups, 1) bytes per row, 8-byte aligned,
 * categorical; 4*d_out bytes per row, 4-byte aligned, Gaussian).  An empty shard (M == 0) may pass NULL outputs and a
 * NULL nvec and still publishes its ack. */
int ktb_mlp_bf16_policy_evaluate_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                        int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                        const void* b2, const void* W3, const void* b3, const int32_t* nvec,
                                        int n_groups, size_t taken_offset, float* log_probs, float* entropy,
                                        void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                        size_t chunk_rows, unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_evaluate_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                               int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                               const void* W2, const void* b2, const void* W3, const void* b3,
                                               const int32_t* nvec, int n_groups, size_t mask_offset,
                                               size_t taken_offset, float* log_probs, float* entropy, void* scratch,
                                               void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                               unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_evaluate_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                              int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                              const void* W2, const void* b2, const void* W3v, const void* b3v,
                                              const int32_t* nvec, int n_groups, size_t taken_offset,
                                              float* log_probs, float* entropy, float* values, void* scratch,
                                              void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                              unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_evaluate_masked_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                     int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                     const void* W2, const void* b2, const void* W3v, const void* b3v,
                                                     const int32_t* nvec, int n_groups, size_t mask_offset,
                                                     size_t taken_offset, float* log_probs, float* entropy,
                                                     float* values, void* scratch, void* ctrl_local,
                                                     void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                     unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_evaluate_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                 int d_in, int d_hidden, int d_out, const void* W1, const void* b1,
                                                 const void* W2, const void* b2, const void* W3, const void* b3,
                                                 const float* log_std, size_t taken_offset, float* log_probs,
                                                 float* entropy, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                                 int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_policy_gaussian_evaluate_value_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M,
                                                       int d_in, int d_hidden, int d_out, const void* W1,
                                                       const void* b1, const void* W2, const void* b2,
                                                       const void* W3v, const void* b3v, const float* log_std,
                                                       size_t taken_offset, float* log_probs, float* entropy,
                                                       float* values, void* scratch, void* ctrl_local,
                                                       void* ctrl_root_peer, int rank, size_t chunk_rows,
                                                       unsigned long long seq, uintptr_t stream);

/* Deterministic actor (TD3, DDPG): tanh(mu) with seeded, clipped Gaussian noise, fused into the head.  ktb_mlp_bf16_policy's
 * arguments up to b3, then (noise, noise_clip, squash, seed, row_base, actions).  It stores no logits and no
 * log-probabilities.
 *   - mu_ij is the bf16-rounded head output (ktb_mlp_bf16_policy's logits), t = tanhf(mu) when squash != 0, mu widened
 *     to fp32 otherwise.
 *   - noise (sigma) != 0: z_ij is the noise of ktb_mlp_bf16_policy_gaussian (Philox word j & 1 of counter
 *     (i, j >> 1, 1), i = row_base + row), n = __fmul_rn(sigma, z) clamped to [-noise_clip, noise_clip] by comparisons,
 *     and t = __fadd_rn(t, n).  noise == 0 draws no Philox word and adds nothing.
 *   - actions[i, j] (fp32 [M, d_out], 4 bytes per column; may be a peer pointer) = t clamped to [-1, 1] by comparisons
 *     when squash != 0, t otherwise.  Exploration is noise = sigma with noise_clip = +inf; TD3's target policy
 *     smoothing is noise = 0.2, noise_clip = 0.5; noise = 0 is the deterministic mode of a squashed (SAC: W3 / b3 the
 *     mean rows) or unsquashed (the Gaussian head's mean, widened) policy.
 *   - IEEE cases: a NaN mu gives a NaN action (comparisons keep it).  mu = +-inf gives t = +-1 when squashed, the
 *     action without noise.  noise = +inf with noise_clip = +inf gives +-1 (the sign of z) when squashed, and +-inf
 *     (NaN where mu is the opposite infinity) unsquashed.
 *     noise_clip = 0 adds a signed zero, so t is unchanged but for the sign of a zero t.
 *   - With squash == 0: noise = 1, noise_clip = +inf gives ktb_mlp_bf16_policy_gaussian's actions with log_std = 0 bit
 *     for bit, and noise = 0 gives ktb_mlp_bf16_policy's logits widened to fp32.
 *   - Checks: every check ktb_mlp_bf16_policy runs first; then, with M > 0, a NULL or not 4-byte aligned actions is
 *     KTB_ERR_ARG and d_out > 256 is KTB_ERR_UNSUPPORTED; then a NaN or negative noise or noise_clip is KTB_ERR_ARG.
 *     The pushed form reads only the observation rows from its staging half (ktb_push_scatter_ce feeds it); an empty
 *     pushed shard (M == 0) may pass NULL actions and still publishes its ack.  Writes stay inside actions[M, d_out],
 *     scratch and stage. */
int ktb_mlp_bf16_policy_deterministic(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                      const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                      const void* b3, float noise, float noise_clip, int squash, uint64_t seed,
                                      uint64_t row_base, float* actions, void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_policy_deterministic_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                             int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                             const void* b2, const void* W3, const void* b3, float noise,
                                             float noise_clip, int squash, uint64_t seed, uint64_t row_base,
                                             float* actions, void* scratch, void* ctrl_local, void* ctrl_root_peer,
                                             int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream);

/* Q(s, a) critics (SAC, TD3, DDPG; Ape-X DPG and R2D2 priorities), forward only, with the actions fed into layer 1
 * beside the observations.  One critic on M rows, the user's nn.Linear(d_in + d_act, d_h) -> ReLU -> nn.Linear(d_h,
 * d_h) -> ReLU -> nn.Linear(d_h, 1) over torch.cat([obs, act.to(torch.bfloat16)], -1):
 *     x = [obs | bf16(act)]                     obs bf16 [M, d_in], act fp32 [M, d_act]
 *     h = relu(x W1ᵀ + b1), h = relu(h W2ᵀ + b2), q = fp32(h W3ᵀ + b3)      q fp32 [M]
 *   - Every layer follows ktb_mlp_bf16_policy's rules: the bias joins the fp32 accumulator, each layer rounds once to
 *     bf16, ReLU keeps NaN as torch.relu does (so a NaN action gives a NaN q, and an infinite one a NaN q wherever
 *     the torch definition gives one).
 *   - The action is rounded to bf16 once, to nearest even, as .to(torch.bfloat16) does.  q is the bf16 head output
 *     widened exactly.
 *   - W1p is the user's W1 [d_hidden, d_in + d_act] padded with zero columns to [d_hidden, d_in + 64]; layer 1 runs
 *     over K = d_in + 64, its last K block an action tile [rows, 64] (bf16(act), zero past d_act) packed into scratch
 *     per chunk.  So q equals ktb_mlp_bf16_policy's logits at d_out = 1 over x = [obs | bf16(act) | 0] and W1p, widened
 *     to fp32, bit for bit.  d_in is a multiple of 64, d_hidden of 256, and 1 <= d_act <= 64.
 *   - Arguments: ktb_mlp_bf16_policy's, with d_act in place of d_out, W1p for W1, W3 [1, d_hidden] and b3 [1], then
 *     act (act_offset, a byte offset into the rank's staging half, in the pushed forms) and q.  The _twin entries run
 *     two independent critics on the same (obs, act), the second's (W1p, b1, W2, b2, W3, b3) after the first's, and
 *     store q1, q2 and q_min = q2 < q1 ? q2 : q1, NaN when either is (payload unspecified); a tie gives q1, signed
 *     zeros included, as torch.minimum(q1, q2) does on 0-d CPU tensors (its vectorised CPU kernel gives q2 on a tie
 *     of signed zeros).  A zero q is +0 on H100: the tensor cores sum all-zero products to +0 and a −0 bias
 *     adds to it as +0, so no signed-zero tie of q1 and q2 arises from the kernel.  The action tile is packed once
 *     per chunk for both.
 *   - scratch holds ktb_mlp_critic_scratch_bytes(M, d_hidden): the two hidden activations and the action tile.
 *   - act and the outputs may be peer pointers.  The pushed forms read the actions from their one side
 *     (ktb_mlp_bf16_pushed), act: 4*d_act bytes per row, 4-byte aligned, act_offset bytes into the staging half.
 *   - Checks: every check ktb_mlp_bf16_policy runs first, at d_out = 1 (a twin's second weights and biases as the
 *     first's, right after them); then d_act < 1 is KTB_ERR_ARG and d_act > 64 KTB_ERR_UNSUPPORTED; then, with M > 0, a
 *     NULL or not 4-byte aligned act, q, q1, q2 or q_min is KTB_ERR_ARG.  An empty pushed shard (M == 0) may pass NULL
 *     outputs and still publishes its ack.  Writes stay inside the outputs, scratch and stage. */
size_t ktb_mlp_critic_scratch_bytes(size_t M, int d_hidden);
int ktb_mlp_bf16_critic(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act, const void* W1p,
                        const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                        const float* act, float* q, void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_critic_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden,
                               int d_act, const void* W1p, const void* b1, const void* W2, const void* b2,
                               const void* W3, const void* b3, size_t act_offset, float* q, void* scratch,
                               void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                               unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_critic_twin(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act, const void* W1p,
                             const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                             const void* W1p_2, const void* b1_2, const void* W2_2, const void* b2_2,
                             const void* W3_2, const void* b3_2, const float* act, float* q1, float* q2, float* q_min,
                             void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_critic_twin_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                    int d_hidden, int d_act, const void* W1p, const void* b1, const void* W2,
                                    const void* b2, const void* W3, const void* b3, const void* W1p_2,
                                    const void* b1_2, const void* W2_2, const void* b2_2, const void* W3_2,
                                    const void* b3_2, size_t act_offset, float* q1, float* q2, float* q_min,
                                    void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank, size_t chunk_rows,
                                    unsigned long long seq, uintptr_t stream);

/* TD targets of TD3, DDPG and SAC in one call, forward only: the next actions of an actor, the target critics over
 * them and the Bellman target.  For rows next_obs (bf16 [M, d_in]) with reward and done (fp32 [M]):
 *   - Next action.  _deterministic (TD3, DDPG): a = ktb_mlp_bf16_policy_deterministic's actions, with its noise,
 *     noise_clip, squash, seed and row_base (noise over global rows row_base + i).  _gaussian (SAC): (a, logp) =
 *     ktb_mlp_bf16_policy_gaussian_state's actions and log-probabilities, with its interleaved head aW3s / ab3s,
 *     log_std_min / log_std_max, squash, seed and row_base (the same Philox stream).  The actor is
 *     (aW1, ab1, aW2, ab2, aW3, ab3) with its own d_hidden_actor, which may differ from the critics' d_hidden.
 *   - Critics.  q1 (and q2 with a twin) are ktb_mlp_bf16_critic(_twin)'s values over a, which reaches layer 1 as the
 *     same bf16 action tile.  t = q_min with a twin (its tie and NaN rule) and t = q1 without one (DDPG).
 *   - SAC: t = __fsub_rn(t, __fmul_rn(alpha, logp)).  There is no alpha term in the _deterministic entries.
 *   - y[i] = __fadd_rn(r, __fmul_rn(__fmul_rn(gamma, __fsub_rn(1.f, d)), t)), fp32 [M] (may be a peer pointer): the
 *     evaluation order of reward + gamma * (1 - done) * (t - alpha * logp) on fp32 torch tensors with Python-float
 *     gamma and alpha, which torch rounds to fp32 first.  No FMA contraction.  IEEE cases follow the formula: an
 *     infinite or NaN t gives NaN where gamma * (1 - d) is 0 (done = 1, or gamma = 0), and +-inf or NaN otherwise;
 *     alpha = 0 with an infinite logp gives NaN; a NaN reward or done gives NaN.
 *   - Arguments: ktb_mlp_bf16_critic's up to b3 (W1p [d_hidden, d_in + 64], 1 <= d_act <= 64), the second critic's
 *     (W1p_2, b1_2, W2_2, b2_2, W3_2, b3_2) (all six NULL: a single critic), then d_hidden_actor and the actor's six
 *     pointers, then the policy's arguments in the order of the standalone entry, then reward, done (reward_offset,
 *     done_offset: byte offsets into the rank's staging half, in the pushed forms), gamma, alpha (_gaussian only), y,
 *     then scratch and stage (or the push arguments) and stream.  scratch holds ktb_mlp_td_target_scratch_bytes(M,
 *     d_hidden_actor, d_hidden, d_act): the two hidden activations at the wider d_hidden, the action tile, and the
 *     chunk's fp32 actions, log-probabilities and q1.  No M-sized intermediate is written.
 *   - Checks, in this order: every check of ktb_mlp_bf16_critic (_twin with a second critic; a second critic with a NULL
 *     W1p_2 and another of its six pointers non-NULL is KTB_ERR_ARG there) but those of act and the Q outputs; then
 *     every check of the actor's standalone entry at d_out = d_act and d_hidden_actor, its noise and noise_clip or its
 *     log_std bounds included (the actor and the critics share d_in and d_act, one argument each); then a non-finite
 *     gamma or alpha is KTB_ERR_ARG; then, with M > 0, a NULL or not 4-byte aligned reward, done (pull forms) or y is
 *     KTB_ERR_ARG.  An empty pushed shard (M == 0) may pass NULL outputs and still publishes its ack.  The pushed forms
 *     read reward and done from their two sides (ktb_mlp_bf16_pushed): reward, then done, each fp32, 4 bytes per row,
 *     4-byte aligned.  Writes stay inside y, scratch and stage. */
size_t ktb_mlp_td_target_scratch_bytes(size_t M, int d_hidden_actor, int d_hidden, int d_act);
int ktb_mlp_bf16_td_target_deterministic(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act,
                                         const void* W1p, const void* b1, const void* W2, const void* b2,
                                         const void* W3, const void* b3, const void* W1p_2, const void* b1_2,
                                         const void* W2_2, const void* b2_2, const void* W3_2, const void* b3_2,
                                         int d_hidden_actor, const void* aW1, const void* ab1, const void* aW2,
                                         const void* ab2, const void* aW3, const void* ab3, float noise,
                                         float noise_clip, int squash, uint64_t seed, uint64_t row_base,
                                         const float* reward, const float* done, float gamma, float* y, void* scratch,
                                         void* stage, uintptr_t stream);
int ktb_mlp_bf16_td_target_deterministic_pushed(
    int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_act,
    const void* W1p, const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
    const void* W1p_2, const void* b1_2, const void* W2_2, const void* b2_2, const void* W3_2, const void* b3_2,
    int d_hidden_actor, const void* aW1, const void* ab1, const void* aW2, const void* ab2, const void* aW3,
    const void* ab3, float noise, float noise_clip, int squash, uint64_t seed, uint64_t row_base,
    size_t reward_offset, size_t done_offset, float gamma, float* y, void* scratch, void* ctrl_local,
    void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream);
int ktb_mlp_bf16_td_target_gaussian(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_act,
                                    const void* W1p, const void* b1, const void* W2, const void* b2, const void* W3,
                                    const void* b3, const void* W1p_2, const void* b1_2, const void* W2_2,
                                    const void* b2_2, const void* W3_2, const void* b3_2, int d_hidden_actor,
                                    const void* aW1, const void* ab1, const void* aW2, const void* ab2,
                                    const void* aW3s, const void* ab3s, float log_std_min, float log_std_max,
                                    int squash, uint64_t seed, uint64_t row_base, const float* reward,
                                    const float* done, float gamma, float alpha, float* y, void* scratch, void* stage,
                                    uintptr_t stream);
int ktb_mlp_bf16_td_target_gaussian_pushed(
    int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in, int d_hidden, int d_act,
    const void* W1p, const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
    const void* W1p_2, const void* b1_2, const void* W2_2, const void* b2_2, const void* W3_2, const void* b3_2,
    int d_hidden_actor, const void* aW1, const void* ab1, const void* aW2, const void* ab2, const void* aW3s,
    const void* ab3s, float log_std_min, float log_std_max, int squash, uint64_t seed, uint64_t row_base,
    size_t reward_offset, size_t done_offset, float gamma, float alpha, float* y, void* scratch, void* ctrl_local,
    void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq, uintptr_t stream);

/* DQN and Double DQN targets in one call, forward only: the greedy next action, the target network's Q at it and the
 * Bellman target.  For rows next_obs (bf16 [M, d_in]) with reward and done (fp32 [M]), the target Q-network (W1, b1,
 * W2, b2, W3, b3) and, for Double DQN, an online Q-network (oW1, ob1, oW2, ob2, oW3, ob3) of the same d_in, d_hidden
 * and d_out:
 *   - Qt and Qo are the bf16 logits ktb_mlp_bf16_policy computes for the target and the online network.
 *   - The selector S is Qo with an online network (Double DQN) and Qt without one (DQN); the _masked entries rank
 *     S.masked_fill(~legal, -inf) with the legal-action mask of the next states (uint8 [M, d_out], nonzero: legal).
 *   - a*[i] = torch.argmax(S[i]) with the greedy entries' rules (ties to the lowest column, the first NaN wins, -0 equals
 *     +0, a row whose ranked values are all -inf or that has no legal column gets 0): bit for bit the actions of
 *     ktb_mlp_bf16_policy(_masked) on the selecting network.
 *   - q[i] = fp32(Qt[i, a*[i]]), read from the UNMASKED target logits and widened exactly.  A terminal next state
 *     often has no legal action, and there done = 1: the unmasked read gives Qt[i, 0] and y = r exactly, where a masked
 *     one would give 0 * -inf = NaN.
 *   - y[i] = __fadd_rn(r, __fmul_rn(__fmul_rn(gamma, __fsub_rn(1.f, d)), q)), fp32 [M] (may be a peer pointer): the TD
 *     targets' expression and rounding, no FMA contraction.  IEEE cases follow: a NaN in the selector picks that
 *     column (DQN's y is then NaN; Double DQN's is the target's value there), and an infinite q with done = 1 or with
 *     gamma = 0 gives NaN.  Nothing is drawn, so y does not depend on the chunk size, the form or the rank split, and
 *     DQN's y equals Double DQN's with online = target bit for bit.
 *   - Per row chunk on one stream: Double DQN runs the online network with the greedy head (actions only) into chunk
 *     scratch, then the target network, whose head reads a* there; DQN runs the target network alone.  scratch holds
 *     ktb_mlp_dqn_target_scratch_bytes(M, d_hidden): the two hidden activations and the chunk's int64 a*.  No M-sized
 *     intermediate is written.
 *   - Arguments: ktb_mlp_bf16_policy's up to b3 (the target network), the online network's six pointers (all six NULL:
 *     DQN), mask (the _masked entries), reward, done (rd_offset in the pushed forms), gamma, y, then scratch and stage
 *     (or the push arguments) and stream.
 *   - Checks, in this order: every check of ktb_mlp_bf16_policy (_masked) on the target network, d_out > 256 being
 *     KTB_ERR_UNSUPPORTED; then the online network's pointers and alignment, checked as a twin critic's second (a NULL
 *     oW1 with another of its six pointers non-NULL is KTB_ERR_ARG); then a non-finite gamma is KTB_ERR_ARG; then, with
 *     M > 0, a NULL or not 4-byte aligned reward, done (pull forms) or y is KTB_ERR_ARG.  An empty pushed shard
 *     (M == 0) may pass NULL outputs and still publishes its ack.  The pushed forms read (mask, then) rd from their
 *     sides (ktb_mlp_bf16_pushed): mask d_out bytes per row, and rd one side of interleaved fp32 (reward, done) pairs,
 *     8 bytes per row, 8-byte aligned (the kernel reads reward[2i] and done[2i] there).  Writes stay inside y[M],
 *     scratch and stage. */
size_t ktb_mlp_dqn_target_scratch_bytes(size_t M, int d_hidden);
int ktb_mlp_bf16_dqn_target(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out, const void* W1,
                            const void* b1, const void* W2, const void* b2, const void* W3, const void* b3,
                            const void* oW1, const void* ob1, const void* oW2, const void* ob2, const void* oW3,
                            const void* ob3, const float* reward, const float* done, float gamma, float* y,
                            void* scratch, void* stage, uintptr_t stream);
int ktb_mlp_bf16_dqn_target_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                   int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                   const void* b2, const void* W3, const void* b3, const void* oW1, const void* ob1,
                                   const void* oW2, const void* ob2, const void* oW3, const void* ob3,
                                   size_t rd_offset, float gamma, float* y, void* scratch, void* ctrl_local,
                                   void* ctrl_root_peer, int rank, size_t chunk_rows, unsigned long long seq,
                                   uintptr_t stream);
int ktb_mlp_bf16_dqn_target_masked(int dev, const void* obs, size_t M, int d_in, int d_hidden, int d_out,
                                   const void* W1, const void* b1, const void* W2, const void* b2, const void* W3,
                                   const void* b3, const void* oW1, const void* ob1, const void* oW2, const void* ob2,
                                   const void* oW3, const void* ob3, const uint8_t* mask, const float* reward,
                                   const float* done, float gamma, float* y, void* scratch, void* stage,
                                   uintptr_t stream);
int ktb_mlp_bf16_dqn_target_masked_pushed(int dev, const void* stage_local, size_t stage_stride, size_t M, int d_in,
                                          int d_hidden, int d_out, const void* W1, const void* b1, const void* W2,
                                          const void* b2, const void* W3, const void* b3, const void* oW1,
                                          const void* ob1, const void* oW2, const void* ob2, const void* oW3,
                                          const void* ob3, size_t mask_offset, size_t rd_offset, float gamma, float* y,
                                          void* scratch, void* ctrl_local, void* ctrl_root_peer, int rank,
                                          size_t chunk_rows, unsigned long long seq, uintptr_t stream);

/* ---- generalized advantage estimation (PPO's learner target) --------------------------------------------------------
 *
 * Env-major fp32 [N, T]: row i is environment i's trajectory and column t is step t.  dones[i, t] is the done flag of
 * transition t (the episode ended after the action at step t); last_values[i] is V(s_T), which bootstraps step T - 1.
 * CleanRL's and SB3's `dones[t]` / `episode_starts[t]` mark that observation t STARTS an episode: their transition-t
 * flag is dones[t + 1] (next_done at the last step).
 *
 * Per row, as fp32 operations each rounded to nearest even, with no FMA contraction, starting from acc = 0 and
 * nv = last_values[i], for t = T - 1 down to 0 (r, v, d = rewards, values, dones at [i, t]):
 *     nt    = 1 - d
 *     delta = (r + (gamma * nv) * nt) - v
 *     acc   = delta + (gamma_lam * nt) * acc
 *     adv[i, t] = acc
 *     ret[i, t] = acc + v
 *     nv    = v
 * which is bit for bit the torch loop of tests/policy_gae_cases.py (CleanRL's expression order) when gamma is the
 * fp32 rounding of γ and gamma_lam the fp32 rounding of the double product γ·λ.  A done step multiplies by nt = 0, it
 * does not select: an infinite value or advantage after an episode boundary makes the advantages before it NaN, as in
 * the torch loop.  Rows are independent; the recurrence along a row is evaluated sequentially (no parallel-in-time
 * scan, which would change the bits).
 *
 * Checks, in this order: an unregistered dev is KTB_ERR_STATE; a non-finite gamma or gamma_lam is KTB_ERR_ARG;
 * N·T == 0 is KTB_OK with nothing enqueued (the pointers may then be NULL); otherwise a NULL or not 4-byte-aligned
 * pointer, N·T·4 past SIZE_MAX, or an adv or ret range that overlaps an input range or the other output is
 * KTB_ERR_ARG.  The kernel reads each input element once and writes adv[0, N·T) and ret[0, N·T) once each. */
int ktb_gae_f32(int dev, const float* rewards, const float* values, const float* dones, const float* last_values,
                size_t N, size_t T, float gamma, float gamma_lam, float* adv, float* ret, uintptr_t stream);

/* ---- V-trace (IMPALA's off-policy learner target) -------------------------------------------------------------------
 *
 * Env-major fp32 [N, T] as for ktb_gae_f32: log_rhos[i, t] = log π(a_t|s_t) − log μ(a_t|s_t), the target policy's
 * log-probability of the taken action less the behaviour policy's; dones[i, t] the done flag of transition t;
 * bootstrap[i] = V(s_T).  rho_bar, c_bar and pg_rho_bar are the clipping thresholds ρ̄, c̄ and the policy gradient's
 * ρ̄; +inf means no clip.
 *
 * Per row, as fp32 operations each rounded to nearest even, with no FMA contraction, starting from acc = 0 and
 * nv = nvs = bootstrap[i], for t = T - 1 down to 0 (lr, r, v, d = log_rhos, rewards, values, dones at [i, t]):
 *     rho   = expf(lr)
 *     disc  = gamma * (1 - d)
 *     cr    = rho > rho_bar ? rho_bar : rho
 *     c     = lam * (rho > c_bar ? c_bar : rho)
 *     pr    = rho > pg_rho_bar ? pg_rho_bar : rho
 *     delta = cr * ((r + disc * nv) - v)
 *     acc   = delta + (disc * c) * acc
 *     vs[i, t]     = acc + v
 *     pg_adv[i, t] = pr * ((r + disc * nvs) - v)
 *     nv    = v
 *     nvs   = vs[i, t]
 * which is bit for bit TorchBeast's from_importance_weights made env-major (tests/policy_vtrace_cases.py) when every
 * scalar is the fp32 rounding of its Python value, expf is CUDA's correctly-rounded-to-2-ulp expf without fast math
 * (torch's exp of an fp32 CUDA tensor), and λ = 1 gives TorchBeast's bits.  The clips are compares, so a NaN ρ stays
 * NaN as under torch.clamp.  A done multiplies by 1 - d = 0, it does not select: an infinite value after an episode
 * boundary makes the targets before it NaN, as in the torch loop.  vs[i, t + 1] is the scan's previous result, so one
 * backward pass produces both outputs.
 *
 * Checks, in this order: an unregistered dev is KTB_ERR_STATE; a non-finite gamma or lam, or a NaN or non-positive
 * rho_bar, c_bar or pg_rho_bar (+inf is allowed) is KTB_ERR_ARG; N·T == 0 is KTB_OK with nothing enqueued (the pointers
 * may then be NULL); otherwise a NULL or not 4-byte-aligned pointer, N·T·4 past SIZE_MAX, or a vs or pg_adv range that
 * overlaps an input range or the other output is KTB_ERR_ARG.  The kernel reads each input element once and writes
 * vs[0, N·T) and pg_adv[0, N·T) once each: 24·N·T + 4·N bytes. */
int ktb_vtrace_f32(int dev, const float* log_rhos, const float* rewards, const float* values, const float* dones,
                   const float* bootstrap, size_t N, size_t T, float gamma, float lam, float rho_bar, float c_bar,
                   float pg_rho_bar, float* vs, float* pg_adv, uintptr_t stream);

/* ---- n-step bootstrapped returns (Ape-X's, R2D2's and A3C's learner targets) ----------------------------------------
 *
 * Env-major fp32 [N, T] as for ktb_gae_f32: dones[i, t] the done flag of transition t; values[i, t] the bootstrap
 * value of state s_t (V(s_t), max_a Q(s_t, a) or a Double-DQN value); baseline[i, t] what the TD error is taken
 * against (Q(s_t, a_t) for Ape-X priorities, values itself for A3C's advantages); last_values[i] = V(s_T).
 *
 * Per element (i, t), as fp32 operations each rounded to nearest even, with no FMA contraction:
 *     acc = t + n < T ? values[i, t + n] : last_values[i]
 *     for k = n - 1 down to 0:
 *         (r, disc) = t + k < T ? (rewards[i, t + k], gamma * (1 - dones[i, t + k])) : (0, 1)
 *         acc = r + disc * acc
 *     ret[i, t] = acc
 *     td[i, t]  = acc - baseline[i, t]
 * which is bit for bit rlax's n_step_bootstrapped_returns at lambda_t = 1 made env-major (tests/policy_nstep_cases.py,
 * the body pads the rollout's end with n - 1 steps of reward 0, discount 1 and value V(s_T)) when gamma is the fp32
 * rounding of γ, as torch rounds a Python scalar that meets an fp32 tensor.  The padded steps past T are real
 * operations, 0 + 1·acc: a −0 becomes +0 there and a NaN stays NaN, as in the padded torch loop.  A done multiplies by
 * 1 - d = 0, it does not select: an infinite bootstrap value after an episode boundary makes the returns before it NaN,
 * as in GAE.  n is at most 32, so every window lies inside the current 32-step tile and the next one; n >= T is
 * allowed, and then every return bootstraps from last_values.  Inputs may alias one another.
 *
 * Checks, in this order: an unregistered dev is KTB_ERR_STATE; n outside [1, 32] or a non-finite gamma is KTB_ERR_ARG;
 * N·T == 0 is KTB_OK with nothing enqueued (the pointers may then be NULL); otherwise a NULL or not 4-byte-aligned
 * pointer, N·T·4 past SIZE_MAX, a ret or td range that overlaps an input range or the other output, or more than
 * 32·(2³¹ − 1) rows is KTB_ERR_ARG.  The kernel reads each input element once (the halo of the last 32-step tile of
 * each warp's span, at most n steps per row, once more) and writes ret[0, N·T) and td[0, N·T) once each: 24·N·T + 4·N
 * bytes. */
int ktb_nstep_f32(int dev, const float* rewards, const float* values, const float* dones, const float* baseline,
                  const float* last_values, size_t N, size_t T, int n, float gamma, float* ret, float* td,
                  uintptr_t stream);

/* ---- Retrace(λ) (the off-policy Q-value target of ACER, Reactor, MPO and Q(λ)) --------------------------------------
 *
 * Env-major fp32 [N, T] as for ktb_gae_f32: log_rhos[i, t] = log π(a_t|s_t) − log μ(a_t|s_t), the target policy's
 * log-probability of the taken action less the behaviour policy's; q[i, t] = Q_target(s_t, a_t); values[i, t] =
 * E_{a~π} Q_target(s_t, a) (max_a Q_target(s_t, a) for a greedy π); dones[i, t] the done flag of transition t;
 * baseline[i, t] what the TD error is taken against, Q_online(s_t, a_t) (it may be q itself); bootstrap[i] =
 * E_π Q_target(s_T, ·).  Columns 0 of log_rhos, q and values are never read.
 *
 * Per row, as fp32 operations each rounded to nearest even, with no FMA contraction, starting from acc = +0, nv =
 * bootstrap[i], nq = −0 and nc = −0, for t = T - 1 down to 0 (lr, r, q, v, d, b = log_rhos, rewards, q, values, dones,
 * baseline at [i, t]):
 *     disc     = gamma * (1 - d)
 *     acc      = r + disc * ((nv - nc * nq) + nc * acc)
 *     ret[i, t] = acc
 *     td[i, t]  = acc - b
 *     nc       = lam * (expf(lr) > 1 ? 1 : expf(lr))
 *     nv       = v
 *     nq       = q
 * which is bit for bit rlax's retrace_continuous made env-major (tests/policy_retrace_cases.py) when gamma and lam are
 * the fp32 roundings of γ and λ, as torch rounds a Python scalar that meets an fp32 tensor, and expf is CUDA's expf
 * without fast math (torch's exp of an fp32 CUDA tensor).  The −0 start values make the general step at t = T − 1 the
 * body's first step, r + disc · bootstrap, bit for bit, a −0 bootstrap included; +0 would give +0 there.  The clip is a
 * compare, so a NaN ρ stays NaN, as under torch.clamp.  A done multiplies by 1 - d = 0, it does not select: an infinite
 * value after an episode boundary makes the targets before it NaN, as in the torch loop.  log_rhos = 0 is Harutyunyan's
 * Q(λ) (c = λ); log_rhos = −inf on the actions a greedy π does not take is Watkins' Q(λ) (c = 0 cuts the trace there).
 * Inputs may alias one another.
 *
 * Checks, in this order: an unregistered dev is KTB_ERR_STATE; a non-finite gamma or lam is KTB_ERR_ARG; N·T == 0 is
 * KTB_OK with nothing enqueued (the pointers may then be NULL); otherwise a NULL or not 4-byte-aligned pointer, N·T·4
 * past SIZE_MAX, a ret or td range that overlaps an input range or the other output, or more than 32·(2³¹ − 1) rows is
 * KTB_ERR_ARG.  The kernel reads each input element once and writes ret[0, N·T) and td[0, N·T) once each: 32·N·T + 4·N
 * bytes. */
int ktb_retrace_f32(int dev, const float* log_rhos, const float* rewards, const float* q, const float* values,
                    const float* dones, const float* baseline, const float* bootstrap, size_t N, size_t T, float gamma,
                    float lam, float* ret, float* td, uintptr_t stream);

/* ---- Prioritized experience replay (the proportional sampler of Ape-X, R2D2 and Rainbow) ----------------------------
 *
 * priorities[C] fp32 holds the stored priorities p_i^α of a replay buffer (usually its filled prefix).  Every call is
 * stateless: it builds the sum tree of the priorities and draws from it.
 *
 * ktb_per_sample_f32 draws strata [j0, j0 + rows) of `batch`.  With P = the least power of two >= C and the leaves
 * priorities[0, C) padded with +0 to P, every node is ONE fp32 add of its two children, left + right, in heap order
 * (node 1 the root, node n's children 2n and 2n + 1, leaf i node P + i).  tree[max(P, 2)] is fp32 scratch of the
 * caller's, left holding: tree[0] = min(priorities) (NaN if any is NaN), tree[1] = total (the root; priorities[0] when
 * C = 1), and tree[n] for 2 <= n < P the internal node n.  Leaves are not copied.  For stratum j, as fp32 operations each
 * rounded to nearest even, with no FMA contraction (value(n) = tree[n] for n < P, else the padded leaf n − P):
 *     u     = (2·(x >> 9) + 1)·2^-24, x = word 0 of Philox4x32-10(counter = (j mod 2^32, j >> 32, 0, 4),
 *             key = (seed mod 2^32, seed >> 32))                     (kubetorch_b200.sampling.replay_noise)
 *     mass  = ((float)j + u) * (total * (1 / (float)batch))           (1 / batch rounded once to fp32)
 *     n     = 1;  while n < P:  go = mass >= value(2n) && value(2n + 1) > 0
 *                               if go: mass = mass - value(2n);   n = 2n + go
 *     i     = n − P;  indices[j − j0] = i
 *     weights[j − j0] = pw(priorities[i] / total * (float)C, −beta) / pw(tree[0] / total * (float)C, −beta)
 * where pw(x, s) is torch's pow of an fp32 CUDA tensor by a scalar: 1 at s = 0, sqrtf(x) at 0.5, rsqrtf(x) at −0.5,
 * 1 / x at −1, x·x at 2, x·x·x at 3, (float)(1.0 / (double)(x·x)) at −2, powf(x, s) otherwise.  This is bit for bit
 * the body of tests/policy_per_cases.py run on the GPU when beta is the fp32 rounding of β and β is exactly 0.5, 1 or 2
 * wherever its rounding is.  A right child is never entered unless its value is > 0 (a NaN never is), so every index
 * lies in [0, C) whatever the priorities hold; with finite priorities >= 0 and a positive, finite total no zero-priority
 * item is drawn (a total that overflows to inf makes mass inf - inf = NaN wherever a left child is inf, and a NaN mass
 * steps left, into zero priorities too), and indices never decrease from one stratum to the next.  The noise depends on (seed, j) only: every split
 * of the strata into calls gives the same bits.
 *
 * ktb_per_update_f32 writes priorities[indices[b]] = pw(|td[b]| + eps, alpha) in place for b in [0, B), where an index
 * repeated in indices takes its LAST occurrence, deterministically.  An index outside [0, C) is skipped: nothing is
 * written for it (the torch body would raise).  No scratch is needed.
 *
 * Checks, in this order: an unregistered dev is KTB_ERR_STATE; a negative or non-finite beta, or a non-finite alpha or
 * eps, is KTB_ERR_ARG; C outside [1, 2^30], batch or B of 0 or j0 + rows > batch is KTB_ERR_ARG, and batch or B above
 * 8192 KTB_ERR_UNSUPPORTED; rows == 0 is then KTB_OK with nothing enqueued; otherwise a NULL pointer, or one not 4-byte
 * aligned (indices: 8-byte), is KTB_ERR_ARG, and so is any overlap of an output (tree, indices, weights; priorities for
 * the update) with an input or another output.  The draw moves about 4·C + 4·P bytes for the tree and, per stratum,
 * log2(P) dependent pairs of loads, mostly from L2. */
int ktb_per_sample_f32(int dev, const float* priorities, size_t C, size_t batch, size_t j0, size_t rows, uint64_t seed,
                       float beta, float* tree, int64_t* indices, float* weights, uintptr_t stream);
int ktb_per_update_f32(int dev, float* priorities, size_t C, const int64_t* indices, const float* td, size_t B,
                       float alpha, float eps, uintptr_t stream);

#ifdef __cplusplus
}
#endif
#endif /* KTB200_H */
