/*
 * duo_b200.h — C ABI of libduo_b200.so: DuoAttention's mixed-head (retrieval + streaming)
 * attention hot path, hand-written for NVIDIA H100 (sm_90a).
 *
 * Plain C: raw device pointers, integers and a cudaStream_t passed as void*.  No torch types.
 * Every function returns 0 on success or a negative DUO_E* code; the message of the last error
 * on the calling thread is available from duo_last_error_string().  No function throws,
 * none allocates device memory (the caller — PyTorch in the reference — owns all buffers),
 * and all work is enqueued on the given stream (re-entrant per stream).
 *
 * What each entry point replaces in the reference (paths relative to mit-han-lab/duo-attention):
 *
 *   duo_layer_create/destroy  – the per-layer views of DuoAttentionStaticKVCache
 *                               (duo_attn/patch/static_kv_cache.py:60-94) re-laid out head-major;
 *                               also pre-encodes the TMA descriptors of the four cache tensors.
 *   duo_rope_append           – apply_rotary_pos_emb (duo_attn/patch/llama.py:177-184) or
 *                               apply_rope_inplace (duo_attn/patch/flashinfer_utils.py:29-59),
 *                               kv_cache.split_kv + put_full_kv (static_kv_cache.py:252-263,109-125)
 *                               and the torch.cat of cached+new streaming KV (llama.py:385-390);
 *                               for INT4 caches also quantize_int4_with_zero_point_per_group
 *                               (demo/quantize_int4.cu:73-178 via demo/int4_kv.py:261-371).
 *   duo_attention             – the flash_attn_func call pair + torch.cat
 *                               (llama.py:225-267 / :364-421; demo/w8a8kv4_llama.py:229-274),
 *                               both head classes in ONE launch; for INT4 caches the
 *                               dequantize pass (demo/int4_kv.py:373-436) is folded into the K/V load.
 *   duo_stream_commit         – compress_and_replace_streaming_kv (static_kv_cache.py:127-167,
 *                               llama.py:273-290; demo/int4_kv.py:438-492) as a ring advance.
 *   duo_quant_int4 / duo_dequant_int4 – the two kernels of demo/quantize_int4.cu (K1 :73-144,
 *                               K2 :9-42) as stand-alone ops (K2 is test/diagnostic only: the
 *                               product never materialises a dequantised cache).
 */
#ifndef DUO_B200_H
#define DUO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define DUO_API __attribute__((visibility("default")))
#else
#define DUO_API
#endif

#define DUO_OK 0
#define DUO_EINVAL -1     /* bad argument / unsupported shape          */
#define DUO_EOVERFLOW -2  /* KV cache capacity exceeded (ValueError in the reference,
                             static_kv_cache.py:112-115)               */
#define DUO_ECUDA -3      /* CUDA runtime / driver error                */
#define DUO_EWORKSPACE -4 /* workspace too small                        */

/* element type of activations and (for DUO_KV_SAME) of the KV cache */
#define DUO_DT_BF16 0
#define DUO_DT_FP16 1
/* KV cache storage */
#define DUO_KV_SAME 0 /* same dtype as activations                                     */
#define DUO_KV_INT4 1 /* packed u4 + fp16 scale/zero per (token, head); activations fp16 or bf16
                         (bf16: K, V and q must lie within fp16's finite range, see attn_int4.cu) */

/* RoPE flavour of duo_rope_append */
#define DUO_ROPE_NONE 0  /* q/k already rotated                                              */
#define DUO_ROPE_HF 1    /* cos/sin tables in the activation dtype, HF op order (llama.py:177-184):
                            round(round(x*cos) + round(rotate_half(x)*sin)) — bit-exact with torch */
#define DUO_ROPE_FP32 2  /* cos/sin tables in fp32, fp32 math, one rounding (flashinfer semantics,
                            flashinfer_utils.py:29-59, with accurate trig)                  */
#define DUO_ROPE_SKIP_Q 0x100 /* OR-able flag: leave q untouched (it was rotated by an earlier call on the
                                 same buffer); k is still rotated on its way into the caches */

/*
 * Geometry + buffers of ONE decoder layer's KV cache, head-major ("heads first, then tokens"):
 *
 *   full_k/full_v : [batch][n_full  ][full_cap            ][head_dim]   retrieval heads
 *   ring_k/ring_v : [batch][n_stream][sink+recent+stage_cap][head_dim]  streaming heads:
 *                   slots [0,sink) = attention sinks, [sink,sink+recent) = ring of the most recent
 *                   tokens (token p lives in slot sink + (p-sink) % recent), and
 *                   [sink+recent, +stage_cap) = staging area holding the K/V of the chunk being
 *                   processed until duo_stream_commit moves its tail into the ring.
 *   KV heads are in the reference's reordered order: retrieval heads first
 *   (duo_attn/patch/utils.py:6-45); q-head i reads kv-head i / group.
 *
 *   DUO_KV_INT4: the staging area starts at slot round_up(sink+recent, 64) instead of sink+recent (the
 *   slots in between are unused) and full_cap / the ring slot count must be multiples of 8, so that every
 *   64-key tile and its scale/zero rows are 16-byte aligned.
 *   DUO_KV_INT4: the k/v tensors hold head_dim/2 bytes per row (high nibble = even element,
 *   demo/quantize_int4.cu:33-40,137) and *_scale / *_zero are fp16 [batch][heads][slots]
 *   (group_size == head_dim == 128, demo/int4_kv.py:140).
 */
typedef struct duo_layer_desc {
  void* full_k;
  void* full_v;
  void* ring_k;
  void* ring_v;
  void* full_k_scale; /* INT4 only, else NULL */
  void* full_k_zero;
  void* full_v_scale;
  void* full_v_zero;
  void* ring_k_scale;
  void* ring_k_zero;
  void* ring_v_scale;
  void* ring_v_zero;
  int64_t full_cap;  /* token capacity of the retrieval cache          */
  int32_t batch;
  int32_t n_full;    /* retrieval KV heads in this layer (0..n_kv)      */
  int32_t n_stream;  /* streaming KV heads (n_kv - n_full)              */
  int32_t group;     /* q heads per kv head                             */
  int32_t head_dim;  /* must be 128                                     */
  int32_t sink;
  int32_t recent;
  int32_t stage_cap; /* max tokens per call (prefill chunk capacity)    */
  int32_t dtype;     /* DUO_DT_*                                        */
  int32_t kv_format; /* DUO_KV_*                                        */
} duo_layer_desc;

/* Streaming/retrieval cache occupancy BEFORE the call (host integers; the caller advances them,
 * exactly like kv_seq_len_list / streaming_kv_seq_len_list in static_kv_cache.py:44-45).
 *   full_len : tokens in the retrieval cache
 *   total    : tokens seen so far by the streaming heads (== full_len unless evict_last ran)
 *   lo       : oldest token position still valid in the ring (>= sink); ring content is
 *              positions [lo, total) ∩ [sink, ∞), sinks are positions [0, min(total, sink)).   */
typedef struct duo_cache_state {
  int64_t full_len;
  int64_t total;
  int64_t lo;
  /* Optional (may be NULL): device array {full_len, total, lo}.  When set, duo_rope_append, duo_attention (chunks
   * of at most DUO_DECODE_MAX_Q tokens) and duo_stream_commit read the occupancy from DEVICE memory at kernel
   * start, so a captured CUDA graph of a decode step can be replayed while the context grows; the host values
   * above must then be upper-bound-consistent (they size the launch and drive the capacity checks).
   * duo_state_advance moves the device copy forward after a step. */
  const int64_t* device_state;
  /* Sequence sharding of the retrieval heads across tensor-parallel ranks (scope row f1; all zero = off).  With
   * seq_world > 1 the layer's full_k/full_v hold only the block-cyclic slice of rank seq_rank — token position p lives
   * on rank (p / seq_block) % seq_world at local row (p / (seq_block*seq_world)) * seq_block + p % seq_block, so a
   * slice is ordered by position and balanced at any length — while full_len keeps counting GLOBAL tokens (full_cap
   * is the local capacity).  duo_rope_append then appends only the positions this rank owns; duo_attention_seq
   * attends the local slice.  Streaming heads are not sharded.  The reference shards by head only
   * (duo_attn/utils.py:151-179). */
  int32_t seq_rank, seq_world, seq_block, seq_reserved;
} duo_cache_state;

typedef struct duo_layer duo_layer; /* opaque: desc + pre-encoded TMA descriptors (host memory) */

DUO_API int duo_layer_create(const duo_layer_desc* desc, duo_layer** out);
DUO_API void duo_layer_destroy(duo_layer* layer);

/* Bytes of scratch duo_attention needs for this geometry (split-KV partials + arrival counters).
 * The buffer must be zero-initialised once; the kernels leave the counters zeroed.            */
DUO_API size_t duo_workspace_bytes(int32_t batch, int32_t n_kv_heads, int32_t group, int32_t max_q_len);

/*
 * RoPE + KV append for one chunk of q_len tokens (all batch rows).
 *   qkv       : [batch][q_len][(n_q + 2 n_kv) * head_dim] fused projection output, row stride
 *               qkv_row_stride elements; q is rotated IN PLACE, k is rotated on its way into the
 *               caches, v is copied (INT4: both quantised, K1 semantics).
 *   cos, sin  : [q_len][head_dim] tables (dtype per rope_mode), shared by all batch rows.
 * Retrieval heads' K/V go to full_{k,v}[.., full_len + t, :]; streaming heads' K/V go to the
 * staging slots ring_{k,v}[.., sink+recent + t, :].
 * Returns DUO_EOVERFLOW if full_len + q_len > full_cap or q_len > stage_cap.
 */
DUO_API int duo_rope_append(const duo_layer* layer, const duo_cache_state* st, void* qkv, int64_t qkv_row_stride,
                    const void* cos, const void* sin, int32_t rope_mode, int32_t q_len, void* stream);

/*
 * Mixed-head attention for one chunk, both head classes in one launch.  Must follow
 * duo_rope_append for the same chunk and state.
 *   q   : [batch][q_len][n_q][head_dim], token stride q_row_stride elements (the rotated q inside qkv)
 *   out : [batch][q_len][n_q][head_dim] contiguous
 * Retrieval q-heads attend keys [0, full_len + t] (bottom-right causal); streaming q-heads attend
 * the valid sink+ring slots plus staged chunk tokens [0, t].  softmax scale `scale`
 * (1/sqrt(head_dim) in the reference), fp32 softmax, P rounded to the activation dtype before PV.
 * q_len <= DUO_DECODE_MAX_Q uses the split-KV bandwidth kernel, larger chunks the tensor-core
 * prefill kernel.
 */
#define DUO_DECODE_MAX_Q 16
DUO_API int duo_attention(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride,
                  void* out, int32_t q_len, float scale, void* workspace, size_t workspace_bytes,
                  void* stream);

/*
 * One launch for a whole decode-sized chunk (group * q_len <= 16): duo_rope_append + duo_attention +
 * duo_stream_commit fused — RoPE of q in registers, RoPE(k) / v of the new tokens written straight to their final
 * cache rows (retrieval: full_len + t; streaming: sink / ring slot, no staging round trip) and attended from a tile
 * built in shared memory.  Replaces, per decoder layer and decode step, what the reference does in
 * duo_attn/patch/llama.py:347-362 (RoPE), :353-362 + static_kv_cache.py:109-125 (append), :364-421 (attention) and
 * :423-425 + static_kv_cache.py:127-167 (streaming compaction).  `qkv` as for duo_rope_append but NOT modified;
 * cos / sin / rope_mode as for duo_rope_append (no DUO_ROPE_SKIP_Q); rows must be 16-byte aligned.
 * INT4 caches (group * q_len <= DUO_DECODE_MAX_Q_INT4, fp16 or bf16 activations): the K1 quantisation of the new K / V
 * (demo/quantize_int4.cu:73-144, done by the reference in int4_kv.py:261-371 before every attention call) is part of the
 * same launch — the CTA that owns the end of a head's key range rotates and quantises the new rows into the cache, reads
 * them back with the rest of its keys, and commits the streaming ring when it has drained its pipeline; cache content
 * and outputs are bit-identical to duo_rope_append + duo_attention + duo_stream_commit.  The very first chunk of a
 * sequence must still go through the three calls on a 16-bit layer of the activation dtype (DUO_KV_SAME): the
 * reference attends the raw K / V there (demo/w8a8kv4_llama.py:229-238).
 */
#define DUO_DECODE_MAX_Q_INT4 8
DUO_API int duo_decode_fused(const duo_layer* layer, const duo_cache_state* st, const void* qkv, int64_t qkv_row_stride,
                             const void* cos, const void* sin, int32_t rope_mode, void* out, int32_t q_len, float scale,
                             void* workspace, size_t workspace_bytes, void* stream);

/*
 * duo_decode_ragged: duo_decode_fused for a batch whose rows have different lengths, one launch per layer and step.
 * Each row b has its own occupancy, read from DEVICE memory at kernel start (so a captured graph can be replayed
 * while the rows grow at different points):
 *   row_state : device int64 [batch][4] = {full_len, total, lo, flags} per row (semantics of duo_cache_state).
 *               flags bit 0 set (DUO_ROW_IDLE): row b is IDLE and sits out the step: none of its retrieval keys, sink or
 *               ring slots is read, nothing of it is written (no append, no ring commit, its rows of `out` keep what
 *               they held).  The other bits must be 0.  The active rows are partitioned as a compact batch of just
 *               those rows (mean length over them, `want` for their number, slots in row order), unless that batch's
 *               splits would not fit the grid: `want` is then clamped to floor(slots / n_active) - 1.  With every
 *               row active the partition and the bits are those of the all-active launch; with every row idle the
 *               launch writes nothing.
 *   cos / sin : [batch][q_len][head_dim] per-row tables (dtype per rope_mode, as for duo_decode_fused)
 *   qkv / out : as for duo_decode_fused; q_len is the same for every row, group * q_len <= DUO_DECODE_MAX_Q
 *   max_full_len : host upper bound of the rows' full_len, used only for the capacity check
 * For every row: RoPE of q and of the new K, append to retrieval rows full_len[b] + t and to the row's sink / ring
 * slots, both head classes, split-KV with the hierarchical merge, and the ring commit.  Retrieval work is balanced
 * by keys: keys-per-split comes from the mean row length and the ~2 CTAs/SM budget, and row b takes
 * ceil(full_len[b] / keys_per_split) splits, so one long row next to short ones is spread over most of the grid.
 * The grid size depends only on the layer and the device.  With every row at the same length the partition,
 * the outputs and the cache bytes equal duo_decode_fused's at the same batch size.
 * 16-bit KV only (INT4 layers: DUO_EINVAL, see duo_decode_ragged_int4); batch <= DUO_RAGGED_MAX_BATCH (else DUO_EINVAL); DUO_EOVERFLOW if
 * max_full_len + q_len > full_cap.  `workspace` must hold duo_ragged_workspace_bytes(batch, n_kv_heads) bytes,
 * zero-initialised once (DUO_EWORKSPACE otherwise); it may be shared with duo_workspace_bytes() users.
 */
#define DUO_RAGGED_MAX_BATCH 64
#define DUO_ROW_IDLE 1 /* row_state[b][3] bit 0: row b sits out the batched launches (see above) */
DUO_API int duo_decode_ragged(const duo_layer* layer, const int64_t* row_state, int64_t max_full_len, const void* qkv,
                              int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode, void* out,
                              int32_t q_len, float scale, void* workspace, size_t workspace_bytes, void* stream);
/* Workspace bytes of duo_decode_ragged for any layer with n_kv_heads kv heads (every retrieval / streaming split)
 * and this batch on the current device; 0 for a bad argument. */
DUO_API size_t duo_ragged_workspace_bytes(int32_t batch, int32_t n_kv_heads);
/*
 * duo_decode_ragged_int4: duo_decode_ragged on an INT4 layer (fp16 or bf16 activations), one launch per layer and
 * step; same arguments.  Per row it is duo_decode_fused's INT4 step (RoPE of q in registers, RoPE + K1 quantisation of
 * the new K / V into retrieval rows full_len[b] + t by the split whose key range holds them, both head classes, ring
 * commit at the row's own total / lo).  Row b has full_len[b] + q_len keys; keys-per-split follows the INT4 decode
 * policy (128-key tiles, >= 1024 keys per split, ~4 CTAs/SM), so with every row at the same length the partition, the
 * outputs and the cache bytes equal duo_decode_fused's at the same batch size.  Idle rows (row_state flags, see
 * duo_decode_ragged) are skipped as there, with the partition of the INT4 policy.  An active row must not be empty
 * (full_len = total = 0): the first call on a sequence attends the raw 16-bit K / V (see duo_decode_fused).
 * group * q_len <= DUO_DECODE_MAX_Q_INT4, batch <= DUO_RAGGED_MAX_BATCH, INT4 layers only (else DUO_EINVAL);
 * DUO_EOVERFLOW if max_full_len + q_len > full_cap.  `workspace` must hold
 * duo_ragged_int4_workspace_bytes(batch, n_kv_heads) bytes, zero-initialised once.
 */
DUO_API int duo_decode_ragged_int4(const duo_layer* layer, const int64_t* row_state, int64_t max_full_len,
                                   const void* qkv, int64_t qkv_row_stride, const void* cos, const void* sin,
                                   int32_t rope_mode, void* out, int32_t q_len, float scale, void* workspace,
                                   size_t workspace_bytes, void* stream);
/* Workspace bytes of duo_decode_ragged_int4, as duo_ragged_workspace_bytes; 0 for a bad argument. */
DUO_API size_t duo_ragged_int4_workspace_bytes(int32_t batch, int32_t n_kv_heads);
/*
 * Ragged batches with per-row capacities: one retrieval-cache POOL per layer instead of [batch][n_full][full_cap].
 *   duo_layer_create_pooled : `desc` as for a ragged layer (full_cap is not used), except that full_k / full_v (INT4:
 *       also full_{k,v}_{scale,zero}) point at pools of pool_tokens * n_full rows of head_dim elements (INT4:
 *       head_dim / 2 bytes, and one fp16 scale / zero per row).  Row b owns the tokens [first_b, first_b + cap_b) of
 *       the pool; its region is the contiguous block [n_full][cap_b][head_dim] starting at pool row first_b * n_full,
 *       i.e. exactly a batch-1 cache of capacity cap_b (so key j of retrieval head h is pool row
 *       first_b * n_full + h * cap_b + j).  With equal capacities and first_b = b * cap the pool is byte for byte the
 *       [batch][n_full][cap][head_dim] layout.  Streaming rings keep their [batch][n_stream][slots] layout.  16-bit
 *       layers get tensor maps over the pool.  DUO_EINVAL, before any CUDA call, if pool_tokens is not a positive
 *       multiple of 128 or pool_tokens * n_full does not fit a 32-bit TMA coordinate.
 *   duo_decode_ragged_pooled : duo_decode_ragged (16-bit layers, group * q_len <= DUO_DECODE_MAX_Q) or
 *       duo_decode_ragged_int4 (INT4 layers, group * q_len <= DUO_DECODE_MAX_Q_INT4, no empty row) on a pooled layer;
 *       same arguments and workspace, same partition, and the same bits as the uniform-capacity launch at the same
 *       lengths, plus
 *         row_geom : device int64 [batch][2] = {first_b, cap_b} in tokens, read at kernel start (a captured graph keeps
 *                    working after a row moves).  Contract, not checked by the kernel: the regions are disjoint, first_b
 *                    and cap_b are multiples of 128 and first_b + cap_b <= pool_tokens.
 *         min_room : host value min_b (capacity_b - full_len_b) over the active rows; DUO_EOVERFLOW if q_len >
 *                    min_room.
 *       Idle rows (row_state flags, see duo_decode_ragged) are skipped as there, in both formats.
 *       DUO_EINVAL for a handle not created by duo_layer_create_pooled; duo_decode_ragged and duo_decode_ragged_int4
 *       refuse a pooled handle.
 */
DUO_API int duo_layer_create_pooled(const duo_layer_desc* desc, int64_t pool_tokens, duo_layer** out);
DUO_API int duo_decode_ragged_pooled(const duo_layer* layer, const int64_t* row_state, const int64_t* row_geom,
                                     int64_t min_room, const void* qkv, int64_t qkv_row_stride, const void* cos,
                                     const void* sin, int32_t rope_mode, void* out, int32_t q_len, float scale,
                                     void* workspace, size_t workspace_bytes, void* stream);
/*
 * duo_decode_ragged_shared: duo_decode_ragged_pooled for a pooled layer (16-bit or INT4) whose rows may share a prefix: several
 * continuations of one long prompt read the prompt's retrieval keys once per step instead of once per row.  Same
 * arguments, plus
 *   row_share : device int64 [batch][2] = {d, P} per row, read at kernel start like row_geom.  d = -1 (or P = 0): a
 *               plain pooled row.  d = b: row b is a DONOR; its keys stay at their rows j of its region.  d != b: row b
 *               is a SHARER of donor d: its keys j < P are the donor's (rows j of the donor's region), its own keys
 *               j >= P live at row j - P of its own region.  P is a multiple of 128 (no 64-key tile straddles it) and
 *               at most the donor's full_len.  The rows with one {d, P} form a group; a donor names the P of one of its
 *               groups and is a member of that group (its other groups' prefixes are read by their sharers only).
 * Two launches, one after the other on `stream`:
 *   1. prefix: for every group, retrieval head and split of the keys [0, P): the TMA tiles are streamed once for all
 *      the group's members, whose packed query rows (group * q_len per member, q rotated in registers as the fused
 *      decode does) fill the M dimension of the 64-row mma.sync kernel; a group of more than 64 packed rows (16 members
 *      at group 4, q_len 1) takes further 64-row blocks, each of which streams the prefix again.  No causal mask.
 *      Split-KV with the hierarchical merge; the result is fp32 normalised O and the log2-domain log-sum-exp per
 *      (row, token, retrieval q-head) in the workspace.  The grid depends only on the layer and the device.
 *   2. suffix: the pooled ragged decode over every row's own keys [P_b, full_len_b) (all keys for a plain row) plus the
 *      new tokens, with the RoPE, append and ring commit of duo_decode_ragged_pooled; keys-per-split is taken over the
 *      keys this launch reads; the final store folds in the row's prefix partial before rounding.
 * Idle rows (row_state flags, see duo_decode_ragged) are skipped by both launches: a group's members are its active
 * rows, a group whose members are all idle takes no slot, and an idle donor's prefix is still streamed for its active
 * sharers.  With no row sharing, the outputs and cache bytes equal duo_decode_ragged_pooled's.
 * INT4 layers take the INT4 twins of both launches: the prefix launch is the 64-row INT4 kernel (64-key tiles of codes
 * and fp16 scale / zero, dequantised in the load) with the same work items; the suffix launch is the pooled ragged INT4
 * decode (keys-as-M kernel, its key partition taken over the keys it reads), with the same fold.
 * DUO_EINVAL, before any CUDA call: a null pointer, a handle not created by duo_layer_create_pooled, group * q_len outside
 * [1, DUO_DECODE_MAX_Q] (INT4 layers: [1, DUO_DECODE_MAX_Q_INT4]); DUO_EOVERFLOW if q_len > min_room (min_room counts a sharer's capacity as P plus its region);
 * DUO_EWORKSPACE if `workspace` holds fewer than duo_ragged_shared_workspace_bytes(batch, n_kv_heads) bytes
 * (zero-initialised once; it serves duo_decode_ragged_pooled too).
 */
DUO_API int duo_decode_ragged_shared(const duo_layer* layer, const int64_t* row_state, const int64_t* row_geom,
                                     const int64_t* row_share, int64_t min_room, const void* qkv,
                                     int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode,
                                     void* out, int32_t q_len, float scale, void* workspace, size_t workspace_bytes,
                                     void* stream);
/* Workspace bytes of duo_decode_ragged_shared for any layer of either KV format with n_kv_heads kv heads and this batch
 * on the current device; 0 for a bad argument. */
DUO_API size_t duo_ragged_shared_workspace_bytes(int32_t batch, int32_t n_kv_heads);
/*
 * duo_attention_shared: duo_attention for a prefill-sized chunk of a SHARER (a row whose first prefix_len retrieval keys
 * are another row's).  `layer` is the sharer's batch-1 handle (its own region and rings), `prefix` the donor's batch-1
 * handle (its region); `st` is the sharer's logical occupancy (full_len counts the shared keys).  Retrieval q-head t sees
 * keys [0, full_len + t]: key j < prefix_len is row j of the prefix's region, key j >= prefix_len row j - prefix_len of
 * the layer's own region.  Streaming heads are those of duo_attention on `layer`.  Call duo_rope_append on `layer` first
 * with full_len - prefix_len (the new keys land at own rows full_len - prefix_len + t), and duo_stream_commit after.
 * Kernels, tiles and split-KV partition are duo_attention's: the wgmma kernel for q_len >= 128 with sink + recent <=
 * 2048, else the 64-row mma.sync kernel (`workspace` as for duo_attention).  INT4 handles (both): the INT4 kernels of
 * duo_attention, 16-row for 9..16 packed rows and 64-row above, each tile's codes, scale and zero read from the region
 * that holds its keys (duo_attention's dequantised image for chunks >= 128 tokens is the caller's choice, see
 * DuoRaggedINT4KVCache).  Outputs are bit-identical to duo_attention on a row that holds all the keys itself.
 * DUO_EINVAL, before any CUDA call: a null pointer, a pooled handle, handles of different KV formats, device_state or a
 * sequence-shard descriptor in `st`, group * q_len <= DUO_DECODE_MAX_Q (INT4: DUO_DECODE_MAX_Q_INT4; decode-sized chunks:
 * duo_decode_ragged_shared), prefix_len
 * not a positive multiple of 128 or larger than full_len or the prefix's full_cap, handles that disagree on n_full,
 * group, head_dim, dtype or are not batch 1.  DUO_EOVERFLOW if full_len - prefix_len + q_len > layer's full_cap (layers
 * with retrieval heads) or q_len > stage_cap.
 */
DUO_API int duo_attention_shared(const duo_layer* layer, const duo_layer* prefix, int64_t prefix_len,
                                 const duo_cache_state* st, const void* q, int64_t q_row_stride, void* out,
                                 int32_t q_len, float scale, void* workspace, size_t workspace_bytes, void* stream);
/*
 * duo_prefill_ragged: a batched prefill of a ragged batch.  Row b of the 16-bit `layer` (a ragged layer of batch B,
 * uniform or pooled) takes a chunk of lengths[b] >= 0 tokens; the chunks are packed back to back in `qkv` (T = sum of
 * the lengths rows, qkv_row_stride elements apart, 16-byte aligned), row b's from packed token o_b = lengths[0] + ... +
 * lengths[b-1], as in flash_attn_varlen_func.  Rows with lengths[b] == 0 are not touched.  Three launches, whatever B:
 *   1. RoPE + append: packed token o_b + t is rotated with row o_b + t of the packed cos / sin tables ([T][128], as for
 *      duo_rope_append; q is rotated in place); its retrieval K/V go to row full_len_b + t of row b's cache (a sharer's:
 *      own region row full_len_b - P_b + t), its streaming K/V to row b's staging slot sink + recent + t.
 *   2. attention: the wgmma prefill kernel over all rows' chunks, one CTA per (row, 128-row query tile, q-head); each
 *      row attends its own keys with the masks of duo_attention (a sharer's keys j < P_b are the donor's region rows, as
 *      in duo_attention_shared).  out [T][n_q_heads][128].
 *   3. ring commit of every row's staged chunk against its own total.
 * Row b's occupancy {full_len, total, lo} is read from row_state (as for duo_decode_ragged; the flags word is ignored:
 * an idle row with a chunk is prefilled, which is how an idle row is admitted); row_geom {first, cap} of a pooled layer
 * (NULL for a uniform one) and row_share {donor, P} (NULL: nothing shared; pooled layers only) as for
 * duo_decode_ragged_shared.  row_state is not advanced: the caller advances each participating row by its length.
 * For a row with a chunk of >= 128 tokens the outputs and every cache byte are bit-identical to those of duo_rope_append
 * + duo_attention (duo_attention_shared on a sharer) + duo_stream_commit on that row's batch-1 handle; shorter chunks,
 * which duo_attention hands to the mma.sync kernel, agree to rounding.  A chunk of a few tokens over a long context
 * occupies a 128-row tile: decode steps belong to duo_decode_ragged.  `workspace` is not used (may be NULL).
 * lengths and row_room are HOST arrays of B entries (copied into the kernel parameters).  DUO_EINVAL, before any CUDA
 * call: a null pointer (cos / sin only with rope_mode != DUO_ROPE_NONE), an INT4 layer, sink + recent > 2048, batch >
 * DUO_RAGGED_MAX_BATCH, row_geom given for a uniform layer or missing for a pooled one, row_share for a uniform layer, a
 * negative length, a bad rope_mode or unaligned qkv rows.  DUO_EOVERFLOW, before any CUDA call: lengths[b] > row_room[b]
 * (layers with retrieval heads; row_room[b] = row b's capacity minus full_len_b, a sharer's capacity counting P_b) or
 * lengths[b] > stage_cap.  All three kernels are set up before the first is enqueued, so a failed call launches nothing.
 */
DUO_API int duo_prefill_ragged(const duo_layer* layer, const int64_t* row_state, const int64_t* row_geom,
                               const int64_t* row_share, const int32_t* lengths, const int64_t* row_room,
                               const void* qkv, int64_t qkv_row_stride, const void* cos, const void* sin,
                               int32_t rope_mode, void* out, float scale, void* workspace, size_t workspace_bytes,
                               void* stream);
/* row_state[b] += n tokens for every active row b < batch, as duo_state_advance does for one row (one tiny kernel);
 * an idle row (flags bit 0, see duo_decode_ragged) keeps its row_state. */
DUO_API int duo_ragged_state_advance(int64_t* row_state, int32_t batch, int32_t n, int32_t sink, int32_t recent,
                                     void* stream);

/* Diagnostic twin of duo_attention that always takes the mma.sync (bandwidth) kernel family, also for
 * chunk shapes duo_attention hands to the wgmma prefill kernel.  16-bit KV only.  Used by the parity
 * tests to cross-check the two kernel families against each other. */
DUO_API int duo_attention_mma(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride,
                              void* out, int32_t q_len, float scale, void* workspace, size_t workspace_bytes,
                              void* stream);

/* device_state += n tokens: full_len += n, total += n, lo = max(lo, total - recent, sink) (one tiny kernel). */
DUO_API int duo_state_advance(int64_t* device_state, int32_t n, int32_t sink, int32_t recent, void* stream);
/* device_state := {full_len, total, lo}, stream-ordered (the three integers travel as kernel arguments, so repeated
 * evict_last()/clear() calls need no staging buffer and cannot race with earlier copies still in flight). */
DUO_API int duo_state_set(int64_t* device_state, int64_t full_len, int64_t total, int64_t lo, void* stream);

/* Move the tail of the staged chunk into sink/ring slots (call after duo_attention). */
DUO_API int duo_stream_commit(const duo_layer* layer, const duo_cache_state* st, int32_t q_len, void* stream);

/*
 * Stand-alone INT4 group quantisation, group_size == 128 == row length.
 *   in    : fp16 rows, row r at in + r*in_row_stride (elements)
 *   packed: [rows][64] u8, scale/zero: fp16 [rows]
 */
DUO_API int duo_quant_int4(const void* in, int64_t in_row_stride, int64_t rows, void* packed, void* scale,
                   void* zero, void* stream);
DUO_API int duo_dequant_int4(const void* packed, const void* scale, const void* zero, int64_t rows, void* out,
                     void* stream);
/* bf16 image of INT4 rows, for chunks of >= 128 tokens on a bf16 layer (the tensor-core prefill kernel reads 16-bit KV):
 *   out[r][i] = bf16_rn(fmaf(code[r][i], float(scale[r]), float(zero[r])))   (fp32 fma, then one rounding to bf16)
 * packed [rows][64] u8, scale / zero fp16 [rows], out bf16 [rows][128].  duo_dequant_int4 (K2) writes fp16. */
DUO_API int duo_dequant_int4_bf16(const void* packed, const void* scale, const void* zero, int64_t rows, void* out,
                                  void* stream);

/*
 * Caller-side glue between the GEMMs of a decoder layer (the "next" row f3 of the scope table), HF arithmetic:
 *   duo_add_rmsnorm : h = residual + x (if residual != NULL; h is written to out_res if out_res != NULL),
 *                     out_norm = weight * T( h_fp32 * rsqrt(mean(h_fp32^2) + eps) )      [LlamaRMSNorm; replaces
 *                     flashinfer_rmsnorm_forward, duo_attn/patch/flashinfer_utils.py:9-16]
 *   duo_silu_mul    : out = T( T(silu(gate)) * up ) for gate_up = [rows][gate(inter) | up(inter)]
 * rows x hidden / rows x inter, contiguous, hidden and inter multiples of 8.
 */
DUO_API int duo_add_rmsnorm(const void* x, const void* residual, const void* weight, void* out_norm, void* out_res,
                            int64_t rows, int32_t hidden, float eps, int32_t dtype, void* stream);
DUO_API int duo_silu_mul(const void* gate_up, void* out, int64_t rows, int32_t inter, int32_t dtype, void* stream);

/*
 * Building blocks of the sequence-sharded decode (SURVEY.md 8f1, DESIGN.md section 6): a retrieval head's
 * cache is split by position over several layers / ranks; each slice is attended separately and the slices are
 * combined with the online-softmax merge (what flash_attn_func computes over the whole cache in one call,
 * duo_attn/patch/llama.py:393-399, is recovered exactly up to fp32 rounding).
 *   duo_attention_partial : every query row (q as for duo_attention, already rotated, group * q_len <= 16) attends rows
 *       [0, n_keys) of EVERY retrieval head of `layer` (no causal offset, streaming heads are not computed);
 *       out_o  : fp32 [batch][q_len][n_q_heads][128]  normalised output of the slice (retrieval-head rows only)
 *       out_lse: fp32 [batch][q_len][n_q_heads]       log2-domain log-sum-exp: max*scale*log2(e) + log2(sum); -inf
 *                                                      for an empty slice
 *   duo_merge_partials    : out[tok][h][:] = sum_p 2^(lse_p - max) o_p / sum_p 2^(lse_p - max) for h < heads_used;
 *       o_parts fp32 [n_parts][tokens][heads_total][128], lse_parts fp32 [n_parts][tokens][heads_total],
 *       out: activation dtype [tokens][heads_total][128] (rows of heads >= heads_used are left untouched).
 */
DUO_API int duo_attention_partial(const duo_layer* layer, int64_t n_keys, const void* q, int64_t q_row_stride,
                                  float* out_o, float* out_lse, int32_t q_len, float scale, void* workspace,
                                  size_t workspace_bytes, void* stream);
/*
 * duo_attention_seq: one decode-sized chunk (group * q_len <= 16) of the sequence-sharded layout described at
 * duo_cache_state.  Retrieval q-heads attend the local slice (token t sees the local rows of positions
 * <= full_len + t) and report out_o / out_lse exactly as duo_attention_partial does; streaming q-heads (replicated on
 * every rank) are computed normally into `out` ([batch][q_len][n_q][128], rows of retrieval heads untouched).
 * Follow with duo_seq_merge, which exchanges the partials between the ranks and writes the retrieval rows of `out`.
 */
DUO_API int duo_attention_seq(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride,
                              void* out, float* out_o, float* out_lse, int32_t q_len, float scale, void* workspace,
                              size_t workspace_bytes, void* stream);
/*
 * duo_prefill_seq: a prefill-sized chunk (group * q_len > 16, e.g. the next user turn) of the sequence-sharded layout,
 * same arguments and the same partial-output contract as duo_attention_seq (q already rotated and the owned rows
 * already appended by duo_rope_append; follow with the cross-rank merge and duo_stream_commit).  Retrieval q-heads
 * attend the local slice: token t sees the local rows of positions <= full_len + t, so with the slice in position order
 * the chunk is causal inside the slice too; a row that sees no key of the slice gets lse = -inf and O = 0.  Streaming
 * q-heads (replicated) see the ring as it was before the chunk plus the whole chunk causally, exactly as duo_attention,
 * and are written to `out`.  Chunks of >= 128 tokens with sink + recent <= 2048 run on the wgmma prefill kernel (its
 * sequence-shard mode); other chunks on the 64-row mma.sync kernel, which needs `workspace` as duo_attention_seq.
 * 16-bit layers only (an INT4 slice is attended through a 16-bit image of it).  DUO_EINVAL before any CUDA call for a
 * state without a shard descriptor or with device_state, an INT4 layer, a null buffer or a decode-sized chunk
 * (duo_attention_seq); DUO_EOVERFLOW if the rank's slice lacks room for the chunk's positions.
 */
DUO_API int duo_prefill_seq(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride,
                            void* out, float* out_o, float* out_lse, int32_t q_len, float scale, void* workspace,
                            size_t workspace_bytes, void* stream);
/* duo_decode_fused for a sequence-sharded cache, ONE new token per batch row: RoPE + append (by the owner of the position
 * only) + slice attention (partials as duo_attention_seq) + streaming heads + ring commit in one launch; follow with
 * duo_seq_merge. */
DUO_API int duo_decode_fused_seq(const duo_layer* layer, const duo_cache_state* st, const void* qkv, int64_t qkv_row_stride,
                                 const void* cos, const void* sin, int32_t rope_mode, void* out, float* out_o,
                                 float* out_lse, float scale, void* workspace, size_t workspace_bytes, void* stream);
/*
 * duo_decode_fused_seq_shared: duo_decode_fused_seq for FORKS of one sequence-sharded prompt (parallel sampling): batch
 * rows that move in lockstep (one token each per step, one logical length full_len in `st`) and share the first
 * prefix_len = P positions of the prompt.  `prefix` is the donor's batch-1 handle, whose local rows [0, P / world)
 * hold this rank's slice of those positions; `layer` is the forks' batch-B handle over their own slices, which hold
 * the positions p >= P at the rows of a sharded cache of positions p - P (P is a multiple of world * block, so p and
 * p - P have the same owner).  Two launches on `stream`:
 *   1. the prefix rows, streamed once per (retrieval head, 64 packed rows) for the group * B query rows of all forks
 *      (q rotated in registers, no mask, split-KV with the hierarchical merge) into fp32 (O, lse) in the workspace;
 *   2. duo_decode_fused_seq over the own slices with positions shifted by P (the owner of full_len appends the new
 *      token at own row local_index(full_len) - P / world; streaming heads and ring commit unchanged), whose retrieval
 *      CTAs merge the row's prefix partial into the (out_o, out_lse) they store (duo_merge_partials' rule).
 * duo_seq_merge then applies unchanged.  `st` may carry device_state (logical lengths: P is a launch constant).
 * DUO_EINVAL, before any CUDA call: a null pointer; an INT4 or pooled handle; a prefix that is not batch 1; handles
 * that differ in n_full, n_stream, group, head_dim or dtype, or group > 16; no valid sequence-shard descriptor;
 * prefix_len not a positive multiple of world * block, above full_len, or with more local rows than the prefix's
 * full_cap.  DUO_EOVERFLOW if an own slice lacks room for the token; DUO_EWORKSPACE if `workspace` holds fewer than
 * duo_seq_shared_workspace_bytes(batch, n_kv_heads) zero-initialised bytes.
 */
DUO_API int duo_decode_fused_seq_shared(const duo_layer* layer, const duo_layer* prefix, int64_t prefix_len,
                                        const duo_cache_state* st, const void* qkv, int64_t qkv_row_stride,
                                        const void* cos, const void* sin, int32_t rope_mode, void* out, float* out_o,
                                        float* out_lse, float scale, void* workspace, size_t workspace_bytes,
                                        void* stream);
DUO_API size_t duo_seq_shared_workspace_bytes(int32_t batch, int32_t n_kv_heads);
/*
 * duo_prefill_seq_shared: duo_prefill_seq for a prefill-sized chunk (group * q_len > 16, the same q_len on every row)
 * of FORKS of one sequence-sharded prompt, e.g. a different question per fork.  `layer`, `prefix`, prefix_len = P are
 * as for duo_decode_fused_seq_shared; `st` is the forks' LOGICAL occupancy (full_len counts the shared positions) with
 * its shard descriptor.  The rank's slice is the donor's local rows [0, P / world) followed by each fork's own slice:
 * local row j >= P / world is own row j - P / world.  Call duo_rope_append on `layer` first with full_len - P (the new
 * keys land at the own rows of positions p - P), follow with the cross-rank merge and duo_stream_commit (also with
 * full_len - P).  Kernels, tiles, visibility, split-KV partition and outputs are duo_prefill_seq's on a batch-B cache
 * that holds the whole slice in every row, bit for bit: the wgmma kernel for q_len >= 128 with sink + recent <= 2048,
 * else the 64-row mma.sync kernel (`workspace` as for duo_prefill_seq).  The one key tile that straddles P / world is
 * loaded in 8-row pieces from the two sources.
 * DUO_EINVAL, before any CUDA call: a null pointer; an INT4 or pooled handle; a prefix that is not a batch-1 handle of
 * the layer's n_full, n_stream, group, head_dim and dtype; no valid sequence-shard descriptor, or device_state;
 * group * q_len <= 16 (one token per fork: duo_decode_fused_seq_shared); prefix_len not a positive multiple of world *
 * block, above full_len, or with more local rows than the prefix's full_cap; P / world not a multiple of 8.
 * DUO_EOVERFLOW if an own slice lacks room for the chunk (checked with full_len - P) or q_len > stage_cap.
 */
DUO_API int duo_prefill_seq_shared(const duo_layer* layer, const duo_layer* prefix, int64_t prefix_len,
                                   const duo_cache_state* st, const void* q, int64_t q_row_stride, void* out,
                                   float* out_o, float* out_lse, int32_t q_len, float scale, void* workspace,
                                   size_t workspace_bytes, void* stream);
/*
 * The INT4 twins (DUO_KV_INT4 layers only; the 16-bit entry points above refuse INT4 layers), same arguments and same
 * partial-output contract, so duo_seq_merge applies unchanged:
 *   duo_attention_seq_int4: group * q_len <= DUO_DECODE_MAX_Q_INT4; q already rotated and the owned rows already
 *       appended (K1-quantised) by duo_rope_append; follow with duo_seq_merge and duo_stream_commit.
 *   duo_decode_fused_seq_int4: group <= DUO_DECODE_MAX_Q_INT4, ONE token; RoPE + K1 quantisation and append of the new
 *       K / V (by the owner of the position only) + slice attention + streaming heads + ring commit in one launch.
 * A rank whose slice holds no key visible to a row reports lse = -inf and O = 0 for it.  The workspace is the one
 * duo_workspace_bytes() sizes for the layer's (batch, n_kv_heads, group).
 */
DUO_API int duo_attention_seq_int4(const duo_layer* layer, const duo_cache_state* st, const void* q,
                                   int64_t q_row_stride, void* out, float* out_o, float* out_lse, int32_t q_len,
                                   float scale, void* workspace, size_t workspace_bytes, void* stream);
DUO_API int duo_decode_fused_seq_int4(const duo_layer* layer, const duo_cache_state* st, const void* qkv,
                                      int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode,
                                      void* out, float* out_o, float* out_lse, float scale, void* workspace,
                                      size_t workspace_bytes, void* stream);
DUO_API int duo_merge_partials(const float* o_parts, const float* lse_parts, int32_t n_parts, int64_t tokens,
                               int32_t heads_total, int32_t heads_used, void* out, int32_t dtype, void* stream);

/*
 * Head-parallel TP (SURVEY.md 8e / 8f3): the per-layer exchange step of the reference's
 * tensor-parallel sharding (duo_attn/utils.py:174-176, "sum" of the row-parallel o_proj / down_proj partials) as a
 * one-shot all-reduce over NVLink peer memory, fused with the residual add + RMSNorm that consumes it:
 *   out_res  = T( T(sum over ranks of partial) + residual )         (residual may be NULL: no add)
 *   out_norm = weight * T( out_res_fp32 * rsqrt(mean(out_res_fp32^2) + eps) )
 * rows <= max_rows (decode and small chunks; latency-bound sizes).  The caller owns all memory:
 *   data[r]  : rank r's receive buffer, duo_comm_data_bytes() bytes, zero-initialised, mapped on EVERY rank
 *              (CUDA IPC / torch symmetric memory; data[rank] is the local one); 16-byte aligned
 *   flags[r] : rank r's flag words, duo_comm_flag_bytes() bytes, zero-initialised, mapped on every rank
 *   local_state : local device int32[max_rows + 1], zero-initialised (call epochs; last word = error flag,
 *              set to 1 if a peer did not arrive within ~3 s - the result of that call is then undefined)
 * Every rank must issue the same sequence of calls (same rows) on one stream each.  Graph-capturable.
 */
typedef struct duo_comm duo_comm;
typedef struct duo_comm_desc {
  void* data[8];
  void* flags[8];
  void* local_state;
  int32_t rank, world;   /* 2 <= world <= 8 */
  int32_t hidden;        /* row length in elements, multiple of 8, <= 16384 */
  int32_t max_rows;      /* <= 64 */
  int32_t dtype;         /* DUO_DT_* */
} duo_comm_desc;
DUO_API size_t duo_comm_data_bytes(int32_t world, int32_t hidden, int32_t max_rows, int32_t dtype);
DUO_API size_t duo_comm_flag_bytes(int32_t world, int32_t max_rows);
DUO_API int duo_comm_create(const duo_comm_desc* desc, duo_comm** out);
DUO_API void duo_comm_destroy(duo_comm* comm);
DUO_API int duo_allreduce_add_rmsnorm(const duo_comm* comm, const void* partial, const void* residual,
                                      const void* weight, void* out_norm, void* out_res, int32_t rows, float eps,
                                      void* stream);

/*
 * duo_seq_merge: the exchange step of the sequence-sharded decode — one kernel that pushes this rank's (O, lse) partial
 * rows into every rank's receive slots over NVLink peer memory (same push / release-flag / acquire-wait protocol and
 * buffer ownership rules as duo_allreduce_add_rmsnorm), then merges the `world` partials of every row in rank order
 * (bit-identical on all ranks) with the online-softmax rule of duo_merge_partials and writes
 * out[tok][h][:] for h < heads_used in the activation dtype.  tokens * heads_used <= max_rows.
 *   part_o fp32 [tokens][heads_total][128], part_lse fp32 [tokens][heads_total] (as written by duo_attention_seq)
 *   data[r]: duo_seqcomm_data_bytes() bytes, flags[r]: duo_seqcomm_flag_bytes() bytes, zero-initialised, mapped on every
 *   rank; local_state: device int32[max_rows + 1] zero-initialised (epochs; last word = peer-timeout error flag).
 */
typedef struct duo_seqcomm duo_seqcomm;
typedef struct duo_seqcomm_desc {
  void* data[8];
  void* flags[8];
  void* local_state;
  int32_t rank, world;  /* 2 <= world <= 8 */
  int32_t max_rows;     /* <= 512 */
} duo_seqcomm_desc;
DUO_API size_t duo_seqcomm_data_bytes(int32_t world, int32_t max_rows);
DUO_API size_t duo_seqcomm_flag_bytes(int32_t world, int32_t max_rows);
DUO_API int duo_seqcomm_create(const duo_seqcomm_desc* desc, duo_seqcomm** out);
DUO_API void duo_seqcomm_destroy(duo_seqcomm* comm);
DUO_API int duo_seq_merge(const duo_seqcomm* comm, const float* part_o, const float* part_lse, void* out, int32_t tokens,
                          int32_t heads_total, int32_t heads_used, int32_t dtype, void* stream);

DUO_API const char* duo_last_error_string(void);
DUO_API int duo_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DUO_B200_H */
