// C ABI of libduo_b200.so (see include/duo_b200.h).  Thin: argument checks, TMA descriptor
// encoding, dispatch to the launchers.  Never throws, never allocates device memory.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "duo_common.cuh"

namespace duo {

int sm_count_current_device() {
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  int& v = sms[dev & 63];
  if (v == 0) {
    int n = 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 132;
    v = n;
  }
  return v;
}

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
  return DUO_ECUDA;
}

// launchers implemented in the other translation units
size_t mma_workspace_bytes(int batch, int n_kv, int group, int max_q_len);
int launch_attn_mma(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                    int q_len, float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream);
int launch_attn_int4(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                     int q_len, float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream);
bool tc_prefill_supported(const duo_layer* L, const duo_cache_state* st, int q_len);
int launch_attn_tc(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                   int q_len, float scale, cudaStream_t stream);
int launch_attn_tc_seq(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                       float* part_o, float* part_lse, int q_len, float scale, cudaStream_t stream);
int launch_attn_tc_shared(const duo_layer* L, const duo_layer* prefix, long long share_len, const duo_cache_state* st,
                          const void* q, long long q_row_stride, void* out, int q_len, float scale, cudaStream_t stream);
int launch_attn_mma_shared(const duo_layer* L, const duo_layer* prefix, long long share_len, const duo_cache_state* st,
                           const void* q, long long q_row_stride, void* out, int q_len, float scale, void* workspace,
                           size_t workspace_bytes, cudaStream_t stream);
int launch_attn_tc_seq_shared(const duo_layer* L, const duo_layer* prefix, long long prefix_rows,
                              const duo_cache_state* st, const void* q, long long q_row_stride, void* out, float* part_o,
                              float* part_lse, int q_len, float scale, cudaStream_t stream);
int launch_attn_mma_seq_shared(const duo_layer* L, const duo_layer* prefix, long long prefix_rows,
                               const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                               float* part_o, float* part_lse, int q_len, float scale, void* workspace,
                               size_t workspace_bytes, cudaStream_t stream);
int launch_prefill_ragged(const duo_layer* L, const RaggedChunks& rc, void* qkv, long long row_stride, const void* cos,
                          const void* sin, int rope_mode, void* out, float scale, cudaStream_t stream);
int launch_rope_append(const duo_layer* L, const duo_cache_state* st, void* qkv, long long row_stride, const void* cos,
                       const void* sin, int rope_mode, int q_len, cudaStream_t stream);
int launch_stream_commit(const duo_layer* L, const duo_cache_state* st, int q_len, cudaStream_t stream);
int launch_quant_int4(const void* in, long long in_row_stride, long long rows, void* packed, void* scale, void* zero,
                      cudaStream_t stream);
int launch_state_advance(long long* st, int n, int sink, int recent, cudaStream_t stream);
int launch_state_set(long long* st, long long full_len, long long total, long long lo, cudaStream_t stream);
int launch_dequant_int4(const void* packed, const void* scale, const void* zero, long long rows, void* out,
                        cudaStream_t stream);
int launch_dequant_int4_bf16(const void* packed, const void* scale, const void* zero, long long rows, void* out,
                             cudaStream_t stream);

int launch_attn_mma_partial(const duo_layer* L, long long n_keys, const void* q, long long q_row_stride, float* out_o,
                            float* out_lse, int q_len, float scale, void* workspace, size_t workspace_bytes,
                            cudaStream_t stream);
int launch_attn_mma_seq(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                        float* part_o, float* part_lse, int q_len, float scale, void* workspace, size_t workspace_bytes,
                        cudaStream_t stream);
int launch_decode_fused(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                        const void* cos, const void* sin, int rope_mode, void* out, int q_len, float scale,
                        void* workspace, size_t workspace_bytes, cudaStream_t stream);
int launch_decode_fused_int4(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                             const void* cos, const void* sin, int rope_mode, void* out, int q_len, float scale,
                             void* workspace, size_t workspace_bytes, cudaStream_t stream);
int launch_decode_ragged(const duo_layer* L, const long long* row_state, const long long* row_geom, const void* qkv,
                         long long row_stride, const void* cos, const void* sin, int rope_mode, void* out, int q_len,
                         float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream, bool verify = false);
int launch_decode_verify(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                         const void* cos, const void* sin, int rope_mode, void* out, int q_len, float scale,
                         void* workspace, size_t workspace_bytes, cudaStream_t stream);
int launch_attn_mma_verify(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride,
                           void* out, int q_len, float scale, void* workspace, size_t workspace_bytes,
                           cudaStream_t stream);
int launch_stream_commit_ragged(const duo_layer* L, const RaggedChunks& rc, cudaStream_t stream);
size_t ragged_workspace_bytes(int batch, int n_kv);
int launch_decode_ragged_int4(const duo_layer* L, const long long* row_state, const long long* row_geom,
                              const void* qkv, long long row_stride, const void* cos, const void* sin, int rope_mode,
                              void* out, int q_len, float scale, void* workspace, size_t workspace_bytes,
                              cudaStream_t stream);
size_t ragged_int4_workspace_bytes(int batch, int n_kv);
int launch_decode_ragged_shared(const duo_layer* L, const long long* row_state, const long long* row_geom,
                                const long long* row_share, const void* qkv, long long row_stride, const void* cos,
                                const void* sin, int rope_mode, void* out, int q_len, float scale, void* workspace,
                                size_t workspace_bytes, cudaStream_t stream);
size_t ragged_shared_workspace_bytes(int batch, int n_kv);
int launch_decode_ragged_shared_int4(const duo_layer* L, const long long* row_state, const long long* row_geom,
                                     const long long* row_share, const void* qkv, long long row_stride, const void* cos,
                                     const void* sin, int rope_mode, void* out, int q_len, float scale, void* workspace,
                                     size_t workspace_bytes, cudaStream_t stream);
size_t ragged_shared_int4_workspace_bytes(int batch, int n_kv);
int launch_attn_int4_shared(const duo_layer* L, const duo_layer* prefix, long long share_len, const duo_cache_state* st,
                            const void* q, long long q_row_stride, void* out, int q_len, float scale, void* workspace,
                            size_t workspace_bytes, cudaStream_t stream);
int launch_ragged_state_advance(long long* st, int batch, int n, int sink, int recent, cudaStream_t stream);
int launch_decode_fused_seq(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                            const void* cos, const void* sin, int rope_mode, void* out, float* part_o, float* part_lse,
                            float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream);
int launch_decode_fused_seq_shared(const duo_layer* L, const duo_layer* prefix, long long prefix_len,
                                   const duo_cache_state* st, const void* qkv, long long row_stride, const void* cos,
                                   const void* sin, int rope_mode, void* out, float* part_o, float* part_lse, float scale,
                                   void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t seq_shared_workspace_bytes(int batch, int n_kv);
int launch_attn_int4_seq(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride,
                         void* out, float* part_o, float* part_lse, int q_len, float scale, void* workspace,
                         size_t workspace_bytes, cudaStream_t stream);
int launch_decode_fused_seq_int4(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                                 const void* cos, const void* sin, int rope_mode, void* out, float* part_o,
                                 float* part_lse, float scale, void* workspace, size_t workspace_bytes,
                                 cudaStream_t stream);
int launch_merge_partials(const float* o_parts, const float* lse_parts, int n_parts, long long tokens, int heads_total,
                          int heads_used, void* out, int dtype, cudaStream_t stream);
int launch_add_rmsnorm(const void* x, const void* residual, const void* weight, void* out_norm, void* out_res,
                       long long rows, int hidden, float eps, int dtype, cudaStream_t stream);
int launch_silu_mul(const void* gate_up, void* out, long long rows, int inter, int dtype, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// TMA descriptors (cuTensorMapEncodeTiled fetched through the runtime: no -lcuda link dependency)
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
    set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// {head_dim, slots, batch*heads} 16-bit tensor; box {64, box_rows, 1}; 128B swizzle; OOB rows read as zero.
static int encode_kv_map(CUtensorMap* m, void* base, int dtype, long long slots, long long heads, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return DUO_ECUDA;
  cuuint64_t dims[3] = {(cuuint64_t)kHeadDim, (cuuint64_t)slots, (cuuint64_t)heads};
  cuuint64_t strides[2] = {(cuuint64_t)kHeadDim * 2, (cuuint64_t)slots * kHeadDim * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(m, dtype == DUO_DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, base,
                  dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (base=%p slots=%lld heads=%lld)", (int)r, base, slots,
              heads);
    return DUO_ECUDA;
  }
  return DUO_OK;
}

// 8-row-box twins of a 16-bit layer's retrieval maps, for one launch: the pieces of a key tile that straddles the
// donor's and the own rows of a fork's slice (duo_prefill_seq_shared)
int encode_piece_maps(const duo_layer* L, CUtensorMap* k8, CUtensorMap* v8) {
  const duo_layer_desc& d = L->d;
  const long long heads = (long long)d.batch * d.n_full;
  if (int rc = encode_kv_map(k8, d.full_k, d.dtype, d.full_cap, heads, 8)) return rc;
  return encode_kv_map(v8, d.full_v, d.dtype, d.full_cap, heads, 8);
}

// first staging slot of the streaming cache: right after the ring for 16-bit caches (TMA takes any
// coordinate); rounded up to a multiple of 64 for INT4 so that every 64-key tile (and its scale/zero rows)
// starts 16-byte aligned for cp.async.
int stage_offset(const duo_layer_desc& d) {
  const int W = d.sink + d.recent;
  return d.kv_format == DUO_KV_INT4 ? (W + 63) / 64 * 64 : W;
}

}  // namespace duo

using namespace duo;

extern "C" {

const char* duo_last_error_string(void) { return g_err; }
int duo_version(void) { return 100; }

// pool_tokens == 0: a [batch][n_full][full_cap] layer (duo_layer_create); > 0: a pooled ragged layer, whose full_k /
// full_v hold pool_tokens * n_full rows (duo_layer_create_pooled)
static int create_layer(const duo_layer_desc* desc, int64_t pool_tokens, duo_layer** out) {
  *out = nullptr;
  if (desc->head_dim != kHeadDim) {
    set_error("duo_layer_create: head_dim %d unsupported (only 128)", desc->head_dim);
    return DUO_EINVAL;
  }
  if (desc->batch < 1 || desc->n_full < 0 || desc->n_stream < 0 || desc->group < 1 || desc->sink < 0 ||
      desc->recent < 1 || desc->stage_cap < 1 || desc->full_cap < 0) {
    set_error("duo_layer_create: bad geometry");
    return DUO_EINVAL;
  }
  if (desc->dtype != DUO_DT_BF16 && desc->dtype != DUO_DT_FP16) {
    set_error("duo_layer_create: bad dtype %d", desc->dtype);
    return DUO_EINVAL;
  }
  if (desc->kv_format == DUO_KV_INT4) {
    const long long ring_slots = (long long)stage_offset(*desc) + desc->stage_cap;
    if ((pool_tokens == 0 && desc->full_cap % 8 != 0) || ring_slots % 8 != 0) {
      set_error("duo_layer_create: INT4 caches need full_cap and ring slots (%lld) to be multiples of 8", ring_slots);
      return DUO_EINVAL;
    }
  }
  duo_layer* L = new (std::nothrow) duo_layer();
  if (!L) {
    set_error("duo_layer_create: out of host memory");
    return DUO_EINVAL;
  }
  L->d = *desc;
  L->has_full_maps = false;
  L->has_ring_maps = false;
  L->pool_tokens = pool_tokens;
  memset(&L->maps, 0, sizeof(L->maps));
  if (desc->kv_format == DUO_KV_SAME) {
    const long long ring_slots = (long long)desc->sink + desc->recent + desc->stage_cap;
    int rc = DUO_OK;
    // pooled: one {head_dim, pool_tokens * n_full, 1} tensor; rows are addressed through the row coordinate
    const long long slots = pool_tokens ? pool_tokens * desc->n_full : desc->full_cap;
    if (desc->n_full > 0 && slots > 0) {
      const long long heads = pool_tokens ? 1 : (long long)desc->batch * desc->n_full;
      rc = encode_kv_map(&L->maps.full_k64, desc->full_k, desc->dtype, slots, heads, 64);
      if (!rc) rc = encode_kv_map(&L->maps.full_v64, desc->full_v, desc->dtype, slots, heads, 64);
      if (!rc) rc = encode_kv_map(&L->maps.full_k128, desc->full_k, desc->dtype, slots, heads, 128);
      if (!rc) rc = encode_kv_map(&L->maps.full_v128, desc->full_v, desc->dtype, slots, heads, 128);
      L->has_full_maps = (rc == DUO_OK);
    }
    if (!rc && desc->n_stream > 0) {
      const long long heads = (long long)desc->batch * desc->n_stream;
      rc = encode_kv_map(&L->maps.ring_k64, desc->ring_k, desc->dtype, ring_slots, heads, 64);
      if (!rc) rc = encode_kv_map(&L->maps.ring_v64, desc->ring_v, desc->dtype, ring_slots, heads, 64);
      if (!rc) rc = encode_kv_map(&L->maps.ring_k128, desc->ring_k, desc->dtype, ring_slots, heads, 128);
      if (!rc) rc = encode_kv_map(&L->maps.ring_v128, desc->ring_v, desc->dtype, ring_slots, heads, 128);
      L->has_ring_maps = (rc == DUO_OK);
    }
    if (rc) {
      delete L;
      return rc;
    }
  }
  *out = L;
  return DUO_OK;
}

int duo_layer_create(const duo_layer_desc* desc, duo_layer** out) {
  if (!desc || !out) {
    set_error("duo_layer_create: null argument");
    return DUO_EINVAL;
  }
  return create_layer(desc, 0, out);
}

int duo_layer_create_pooled(const duo_layer_desc* desc, int64_t pool_tokens, duo_layer** out) {
  if (!desc || !out) {
    set_error("duo_layer_create_pooled: null argument");
    return DUO_EINVAL;
  }
  *out = nullptr;
  if (pool_tokens < 128 || pool_tokens % 128 != 0) {
    set_error("duo_layer_create_pooled: pool_tokens %lld is not a positive multiple of 128", (long long)pool_tokens);
    return DUO_EINVAL;
  }
  if (desc->n_full > 0 && pool_tokens * desc->n_full > INT32_MAX) {  // (n_full is checked to be >= 0 below)
    set_error("duo_layer_create_pooled: pool of %lld tokens x %d retrieval heads exceeds the 32-bit TMA row coordinate",
              (long long)pool_tokens, desc->n_full);
    return DUO_EINVAL;
  }
  return create_layer(desc, pool_tokens, out);
}

void duo_layer_destroy(duo_layer* layer) { delete layer; }

size_t duo_workspace_bytes(int32_t batch, int32_t n_kv_heads, int32_t group, int32_t max_q_len) {
  return mma_workspace_bytes(batch, n_kv_heads, group, max_q_len);
}

// A sequence-shard descriptor the kernels take: 2..8 ranks, a rank among them, blocks of at least one position.
static bool shard_desc_ok(const duo_cache_state* st) {
  return st->seq_world >= 2 && st->seq_world <= 8 && st->seq_rank >= 0 && st->seq_rank < st->seq_world &&
         st->seq_block >= 1;
}

static int check_chunk(const duo_layer* L, const duo_cache_state* st, int q_len, const char* who) {
  if (!L || !st) {
    set_error("%s: null layer/state", who);
    return DUO_EINVAL;
  }
  if (L->pool_tokens) {
    set_error("%s: a pooled ragged layer is decoded with duo_decode_ragged_pooled only", who);
    return DUO_EINVAL;
  }
  if (q_len < 1) {
    set_error("%s: q_len %d < 1", who, q_len);
    return DUO_EINVAL;
  }
  if (st->full_len < 0 || st->total < 0 || st->lo < 0) {
    set_error("%s: negative cache state", who);
    return DUO_EINVAL;
  }
  long long need = st->full_len + q_len;
  if (st->seq_world != 0) {
    if (!shard_desc_ok(st)) {
      set_error("%s: bad sequence-shard descriptor (rank %d, world %d, block %d)", who, st->seq_rank, st->seq_world,
                st->seq_block);
      return DUO_EINVAL;
    }
    need = seq_local_len(need, st->seq_rank, st->seq_world, st->seq_block);  // rows of this rank's slice after the append
  }
  if (L->d.n_full > 0 && need > L->d.full_cap) {
    set_error("Trying to put %d KVs into a cache with max size %lld, current size: %lld.", q_len,
              (long long)L->d.full_cap, (long long)st->full_len);
    return DUO_EOVERFLOW;
  }
  if (q_len > L->d.stage_cap) {
    set_error("%s: chunk of %d tokens exceeds the staging capacity %d", who, q_len, L->d.stage_cap);
    return DUO_EOVERFLOW;
  }
  return DUO_OK;
}

int duo_rope_append(const duo_layer* layer, const duo_cache_state* st, void* qkv, int64_t qkv_row_stride,
                    const void* cos, const void* sin, int32_t rope_mode, int32_t q_len, void* stream) {
  int rc = check_chunk(layer, st, q_len, "duo_rope_append");
  if (rc) return rc;
  if (!qkv || ((rope_mode & 0xff) != DUO_ROPE_NONE && (!cos || !sin))) {
    set_error("duo_rope_append: null buffer");
    return DUO_EINVAL;
  }
  if ((rope_mode & 0xff) < DUO_ROPE_NONE || (rope_mode & 0xff) > DUO_ROPE_FP32 || (rope_mode & ~(0xff | DUO_ROPE_SKIP_Q))) {
    set_error("duo_rope_append: bad rope_mode %d", rope_mode);
    return DUO_EINVAL;
  }
  if (qkv_row_stride % 4 != 0) {
    set_error("duo_rope_append: row stride must be a multiple of 4 elements");
    return DUO_EINVAL;
  }
  return launch_rope_append(layer, st, qkv, qkv_row_stride, cos, sin, rope_mode, q_len, (cudaStream_t)stream);
}

int duo_attention(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride, void* out,
                  int32_t q_len, float scale, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_chunk(layer, st, q_len, "duo_attention");
  if (rc) return rc;
  if (!q || !out) {
    set_error("duo_attention: null buffer");
    return DUO_EINVAL;
  }
  if (st->seq_world != 0) {
    set_error("duo_attention: sequence-sharded caches are attended with duo_attention_seq");
    return DUO_EINVAL;
  }
  if (layer->d.kv_format == DUO_KV_INT4)
    return launch_attn_int4(layer, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes,
                            (cudaStream_t)stream);
  if (st->device_state && q_len > DUO_DECODE_MAX_Q) {
    set_error("duo_attention: device_state is only supported for chunks of <= %d tokens", DUO_DECODE_MAX_Q);
    return DUO_EINVAL;
  }
  if (tc_prefill_supported(layer, st, q_len))
    return launch_attn_tc(layer, st, q, q_row_stride, out, q_len, scale, (cudaStream_t)stream);
  return launch_attn_mma(layer, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes,
                         (cudaStream_t)stream);
}

int duo_attention_shared(const duo_layer* layer, const duo_layer* prefix, int64_t prefix_len, const duo_cache_state* st,
                         const void* q, int64_t q_row_stride, void* out, int32_t q_len, float scale, void* workspace,
                         size_t workspace_bytes, void* stream) {
  const char* who = "duo_attention_shared";
  if (!layer || !prefix || !st || !q || !out) {
    set_error("%s: null argument", who);
    return DUO_EINVAL;
  }
  if (layer->pool_tokens || prefix->pool_tokens || layer->d.kv_format != prefix->d.kv_format) {
    set_error("%s: batch-1 layers of one KV format only (not pooled)", who);
    return DUO_EINVAL;
  }
  const bool int4 = layer->d.kv_format == DUO_KV_INT4;
  if (st->device_state || st->seq_world != 0) {
    set_error("%s: host occupancy of an unsharded cache only (no device_state, no sequence-shard descriptor)", who);
    return DUO_EINVAL;
  }
  const duo_layer_desc &d = layer->d, &pd = prefix->d;
  if (d.batch != 1 || pd.batch != 1 || d.n_full != pd.n_full || d.group != pd.group || d.head_dim != pd.head_dim ||
      d.dtype != pd.dtype) {
    set_error("%s: the layer and the prefix must be batch-1 handles of one geometry (n_full, group, head_dim, dtype)",
              who);
    return DUO_EINVAL;
  }
  const int max_rows = int4 ? DUO_DECODE_MAX_Q_INT4 : DUO_DECODE_MAX_Q;
  if (q_len < 1 || (long long)d.group * q_len <= max_rows) {
    set_error("%s: chunks of group * q_len > %d rows only (got group %d, q_len %d; decode-sized chunks of a sharer: "
              "duo_decode_ragged_shared)", who, max_rows, d.group, q_len);
    return DUO_EINVAL;
  }
  if (prefix_len <= 0 || prefix_len % 128 != 0 || prefix_len > st->full_len || prefix_len > pd.full_cap) {
    set_error("%s: prefix_len %lld must be a positive multiple of 128 and at most full_len %lld and the prefix's "
              "full_cap %lld", who, (long long)prefix_len, (long long)st->full_len, (long long)pd.full_cap);
    return DUO_EINVAL;
  }
  // the own region holds keys [prefix_len, full_len + q_len) at rows [0, full_len - prefix_len + q_len)
  duo_cache_state own = *st;
  own.full_len = st->full_len - prefix_len;
  if (int rc = check_chunk(layer, &own, q_len, who)) return rc;
  if (int4)
    return launch_attn_int4_shared(layer, prefix, prefix_len, st, q, q_row_stride, out, q_len, scale, workspace,
                                   workspace_bytes, (cudaStream_t)stream);
  if (tc_prefill_supported(layer, st, q_len))
    return launch_attn_tc_shared(layer, prefix, prefix_len, st, q, q_row_stride, out, q_len, scale, (cudaStream_t)stream);
  return launch_attn_mma_shared(layer, prefix, prefix_len, st, q, q_row_stride, out, q_len, scale, workspace,
                                workspace_bytes, (cudaStream_t)stream);
}

// Checks shared by the one-launch decode entry points: the output buffers (`outputs_ok`, checked by the caller), qkv
// and the RoPE tables its rope_mode reads, a known rope_mode, and qkv rows the kernels can load 16 bytes at a time.
static int check_decode_args(const char* who, bool outputs_ok, const void* qkv, int64_t qkv_row_stride, const void* cos,
                             const void* sin, int32_t rope_mode) {
  if (!outputs_ok || !qkv || (rope_mode != DUO_ROPE_NONE && (!cos || !sin))) {
    set_error("%s: null buffer", who);
    return DUO_EINVAL;
  }
  if (rope_mode < DUO_ROPE_NONE || rope_mode > DUO_ROPE_FP32) {
    set_error("%s: bad rope_mode %d", who, rope_mode);
    return DUO_EINVAL;
  }
  if (qkv_row_stride % 8 != 0 || (reinterpret_cast<uintptr_t>(qkv) & 15)) {
    set_error("%s: qkv rows must be 16-byte aligned (row stride a multiple of 8 elements)", who);
    return DUO_EINVAL;
  }
  return DUO_OK;
}

int duo_decode_fused(const duo_layer* layer, const duo_cache_state* st, const void* qkv, int64_t qkv_row_stride,
                     const void* cos, const void* sin, int32_t rope_mode, void* out, int32_t q_len, float scale,
                     void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_chunk(layer, st, q_len, "duo_decode_fused");
  if (!rc) rc = check_decode_args("duo_decode_fused", out != nullptr, qkv, qkv_row_stride, cos, sin, rope_mode);
  if (rc) return rc;
  const int max_rows = layer->d.kv_format == DUO_KV_INT4 ? DUO_DECODE_MAX_Q_INT4 : DUO_DECODE_MAX_Q;
  if (layer->d.group * q_len > max_rows || st->seq_world != 0) {
    set_error("duo_decode_fused: unsharded caches and group * q_len <= %d only (got group %d, q_len %d)", max_rows,
              layer->d.group, q_len);
    return DUO_EINVAL;
  }
  if (layer->d.kv_format == DUO_KV_INT4)
    return launch_decode_fused_int4(layer, st, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, scale, workspace,
                                    workspace_bytes, (cudaStream_t)stream);
  return launch_decode_fused(layer, st, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, scale, workspace,
                             workspace_bytes, (cudaStream_t)stream);
}

size_t duo_ragged_workspace_bytes(int32_t batch, int32_t n_kv_heads) {
  if (batch < 1 || batch > DUO_RAGGED_MAX_BATCH || n_kv_heads < 1) return 0;
  return ragged_workspace_bytes(batch, n_kv_heads);
}

size_t duo_ragged_int4_workspace_bytes(int32_t batch, int32_t n_kv_heads) {
  if (batch < 1 || batch > DUO_RAGGED_MAX_BATCH || n_kv_heads < 1) return 0;
  return ragged_int4_workspace_bytes(batch, n_kv_heads);
}

// Checks shared by the ragged decode entry points after the KV-format check: batch, packed rows (<= max_rows), and the
// capacity of the longest row.
static int check_ragged_rows(const char* who, const duo_layer* layer, int32_t q_len, int max_rows) {
  if (layer->d.batch > DUO_RAGGED_MAX_BATCH) {
    set_error("%s: batch %d exceeds %d rows", who, layer->d.batch, DUO_RAGGED_MAX_BATCH);
    return DUO_EINVAL;
  }
  if (q_len < 1 || layer->d.group * q_len > max_rows) {
    set_error("%s: group * q_len <= %d only (got group %d, q_len %d)", who, max_rows, layer->d.group, q_len);
    return DUO_EINVAL;
  }
  return DUO_OK;
}

static int check_ragged_args(const char* who, const duo_layer* layer, int64_t max_full_len, int32_t q_len,
                             int max_rows) {
  if (int rc = check_ragged_rows(who, layer, q_len, max_rows)) return rc;
  if (max_full_len < 0) {
    set_error("%s: negative max_full_len", who);
    return DUO_EINVAL;
  }
  if (layer->d.n_full > 0 && max_full_len + q_len > layer->d.full_cap) {
    set_error("Trying to put %d KVs into a cache with max size %lld, current size: %lld.", q_len,
              (long long)layer->d.full_cap, (long long)max_full_len);
    return DUO_EOVERFLOW;
  }
  return DUO_OK;
}

// Checks shared by the ragged decode entry points, in this order: their pointers (args_ok), whether the layer has a
// retrieval pool (pooled: the entry point needs one; otherwise it refuses one), the decode arguments.  The pooled entry
// points then check the packed rows and the room of the fullest row (min_room) here; the others check their KV
// format, then check_ragged_args.
static int check_ragged_decode(const char* who, const duo_layer* layer, bool args_ok, bool pooled, const void* qkv,
                               int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode,
                               const void* out, int32_t q_len, int64_t min_room) {
  if (!layer || !args_ok) {
    set_error("%s: null argument", who);
    return DUO_EINVAL;
  }
  if (!pooled && layer->pool_tokens) {
    set_error("%s: a pooled ragged layer is decoded with duo_decode_ragged_pooled", who);
    return DUO_EINVAL;
  }
  if (int rc = check_decode_args(who, out != nullptr, qkv, qkv_row_stride, cos, sin, rope_mode)) return rc;
  if (!pooled) return DUO_OK;
  if (!layer->pool_tokens) {
    set_error("%s: the layer has no retrieval pool (create it with duo_layer_create_pooled)", who);
    return DUO_EINVAL;
  }
  // (INT4: q_len <= 8 <= stage_cap, as for duo_decode_ragged_int4)
  const bool int4 = layer->d.kv_format == DUO_KV_INT4;
  if (int rc = check_ragged_rows(who, layer, q_len, int4 ? DUO_DECODE_MAX_Q_INT4 : DUO_DECODE_MAX_Q)) return rc;
  if (layer->d.n_full > 0 && q_len > min_room) {
    set_error("Trying to put %d KVs into a cache row with room for %lld more (%s).", q_len, (long long)min_room, who);
    return DUO_EOVERFLOW;
  }
  return DUO_OK;
}

// ---- verify chunks (DESIGN §2) ------------------------------------------------------------------------------------
// What every verify entry point refuses after its own checks: INT4 layers, sequence-shard descriptors, more packed rows
// than its kernel holds, and chunks longer than the ring (a token's window would reach past what the ring keeps).
static int check_verify(const char* who, const duo_layer* layer, int32_t seq_world, int32_t q_len, int max_rows) {
  const duo_layer_desc& d = layer->d;
  if (d.kv_format != DUO_KV_SAME) {
    set_error("%s: 16-bit caches only (INT4 caches cannot verify drafts)", who);
    return DUO_EINVAL;
  }
  if (seq_world != 0) {
    set_error("%s: sequence-sharded caches cannot verify drafts", who);
    return DUO_EINVAL;
  }
  if (q_len < 1 || (long long)d.group * q_len > max_rows) {
    set_error("%s: group * q_len <= %d only (got group %d, q_len %d)", who, max_rows, d.group, q_len);
    return DUO_EINVAL;
  }
  if (q_len > d.recent) {
    set_error("%s: a chunk of %d tokens exceeds recent = %d", who, q_len, d.recent);
    return DUO_EINVAL;
  }
  return DUO_OK;
}

int duo_decode_verify(const duo_layer* layer, const duo_cache_state* st, const void* qkv, int64_t qkv_row_stride,
                      const void* cos, const void* sin, int32_t rope_mode, void* out, int32_t q_len, float scale,
                      void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_decode_verify";
  int rc = check_chunk(layer, st, q_len, who);
  if (!rc) rc = check_decode_args(who, out != nullptr, qkv, qkv_row_stride, cos, sin, rope_mode);
  if (!rc) rc = check_verify(who, layer, st->seq_world, q_len, DUO_DECODE_MAX_Q);
  if (rc) return rc;
  return launch_decode_verify(layer, st, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, scale, workspace,
                              workspace_bytes, (cudaStream_t)stream);
}

int duo_attention_verify(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride,
                         void* out, int32_t q_len, float scale, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_attention_verify";
  if (int rc = check_chunk(layer, st, q_len, who)) return rc;
  if (!q || !out) {
    set_error("%s: null buffer", who);
    return DUO_EINVAL;
  }
  if (int rc = check_verify(who, layer, st->seq_world, q_len, DUO_VERIFY_MAX_ROWS)) return rc;
  if (st->device_state && q_len > DUO_DECODE_MAX_Q) {
    set_error("%s: device_state is only supported for chunks of <= %d tokens", who, DUO_DECODE_MAX_Q);
    return DUO_EINVAL;
  }
  return launch_attn_mma_verify(layer, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes,
                                (cudaStream_t)stream);
}

int duo_decode_ragged_verify(const duo_layer* layer, const int64_t* row_state, const int64_t* row_geom,
                             int64_t min_room, const void* qkv, int64_t qkv_row_stride, const void* cos,
                             const void* sin, int32_t rope_mode, void* out, int32_t q_len, float scale,
                             void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_decode_ragged_verify";
  const bool pooled = row_geom != nullptr;
  if (int rc = check_ragged_decode(who, layer, row_state, pooled, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len,
                                   min_room))
    return rc;
  if (int rc = check_verify(who, layer, 0, q_len, DUO_DECODE_MAX_Q)) return rc;
  if (!pooled) {  // (the pooled checks ran in check_ragged_decode)
    if (int rc = check_ragged_rows(who, layer, q_len, DUO_DECODE_MAX_Q)) return rc;
    if (layer->d.n_full > 0 && q_len > min_room) {
      set_error("Trying to put %d KVs into a cache row with room for %lld more (%s).", q_len, (long long)min_room, who);
      return DUO_EOVERFLOW;
    }
  }
  if (q_len > layer->d.stage_cap) {
    set_error("%s: chunk of %d tokens exceeds the staging capacity %d", who, q_len, layer->d.stage_cap);
    return DUO_EOVERFLOW;
  }
  return launch_decode_ragged(layer, reinterpret_cast<const long long*>(row_state),
                              reinterpret_cast<const long long*>(row_geom), qkv, qkv_row_stride, cos, sin, rope_mode, out,
                              q_len, scale, workspace, workspace_bytes, (cudaStream_t)stream, true);
}

int duo_stream_commit_rows(const duo_layer* layer, const int64_t* row_state, const int32_t* counts, void* stream) {
  const char* who = "duo_stream_commit_rows";
  if (!layer || !row_state || !counts) {
    set_error("%s: null argument", who);
    return DUO_EINVAL;
  }
  const duo_layer_desc& d = layer->d;
  if (d.kv_format != DUO_KV_SAME) {
    set_error("%s: 16-bit caches only", who);
    return DUO_EINVAL;
  }
  if (d.batch > DUO_RAGGED_MAX_BATCH) {
    set_error("%s: batch %d exceeds %d rows", who, d.batch, DUO_RAGGED_MAX_BATCH);
    return DUO_EINVAL;
  }
  RaggedChunks rc{};
  rc.row_state = reinterpret_cast<const long long*>(row_state);
  rc.batch = d.batch;
  int n_tok = 0;
  for (int b = 0; b < d.batch; ++b) {
    const int n = counts[b];
    if (n < 0 || n > d.recent) {
      set_error("%s: row %d's count %d outside [0, recent = %d]", who, b, n, d.recent);
      return DUO_EINVAL;
    }
    if (n > d.stage_cap) {
      set_error("%s: row %d's count %d exceeds the staging capacity %d", who, b, n, d.stage_cap);
      return DUO_EOVERFLOW;
    }
    rc.len[b] = n;
    rc.off[b] = n_tok;
    n_tok += n;
  }
  rc.off[d.batch] = n_tok;
  return launch_stream_commit_ragged(layer, rc, (cudaStream_t)stream);
}

int duo_decode_ragged(const duo_layer* layer, const int64_t* row_state, int64_t max_full_len, const void* qkv,
                      int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode, void* out,
                      int32_t q_len, float scale, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_decode_ragged";
  if (int rc = check_ragged_decode(who, layer, row_state, false, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, 0))
    return rc;
  if (layer->d.kv_format != DUO_KV_SAME) {
    set_error("duo_decode_ragged: 16-bit KV only (INT4 caches are decoded with duo_decode_ragged_int4)");
    return DUO_EINVAL;
  }
  if (int rc = check_ragged_args(who, layer, max_full_len, q_len, DUO_DECODE_MAX_Q)) return rc;
  return launch_decode_ragged(layer, reinterpret_cast<const long long*>(row_state), nullptr, qkv, qkv_row_stride, cos,
                              sin, rope_mode, out, q_len, scale, workspace, workspace_bytes, (cudaStream_t)stream);
}

int duo_decode_ragged_int4(const duo_layer* layer, const int64_t* row_state, int64_t max_full_len, const void* qkv,
                           int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode, void* out,
                           int32_t q_len, float scale, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_decode_ragged_int4";
  if (int rc = check_ragged_decode(who, layer, row_state, false, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, 0))
    return rc;
  if (layer->d.kv_format != DUO_KV_INT4) {
    set_error("duo_decode_ragged_int4: INT4 caches only (16-bit caches are decoded with duo_decode_ragged)");
    return DUO_EINVAL;
  }
  // (q_len <= 8 <= stage_cap: duo_layer_create keeps an INT4 layer's staging capacity a multiple of 8)
  if (int rc = check_ragged_args(who, layer, max_full_len, q_len, DUO_DECODE_MAX_Q_INT4)) return rc;
  return launch_decode_ragged_int4(layer, reinterpret_cast<const long long*>(row_state), nullptr, qkv, qkv_row_stride,
                                   cos, sin, rope_mode, out, q_len, scale, workspace, workspace_bytes,
                                   (cudaStream_t)stream);
}

int duo_decode_ragged_pooled(const duo_layer* layer, const int64_t* row_state, const int64_t* row_geom,
                             int64_t min_room, const void* qkv, int64_t qkv_row_stride, const void* cos,
                             const void* sin, int32_t rope_mode, void* out, int32_t q_len, float scale,
                             void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_ragged_decode("duo_decode_ragged_pooled", layer, row_state && row_geom, true, qkv, qkv_row_stride,
                                   cos, sin, rope_mode, out, q_len, min_room))
    return rc;
  const long long* rs = reinterpret_cast<const long long*>(row_state);
  const long long* rg = reinterpret_cast<const long long*>(row_geom);
  if (layer->d.kv_format == DUO_KV_INT4)
    return launch_decode_ragged_int4(layer, rs, rg, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, scale,
                                     workspace, workspace_bytes, (cudaStream_t)stream);
  return launch_decode_ragged(layer, rs, rg, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, scale, workspace,
                              workspace_bytes, (cudaStream_t)stream);
}

int duo_decode_ragged_shared(const duo_layer* layer, const int64_t* row_state, const int64_t* row_geom,
                             const int64_t* row_share, int64_t min_room, const void* qkv, int64_t qkv_row_stride,
                             const void* cos, const void* sin, int32_t rope_mode, void* out, int32_t q_len, float scale,
                             void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_ragged_decode("duo_decode_ragged_shared", layer, row_state && row_geom && row_share, true, qkv,
                                   qkv_row_stride, cos, sin, rope_mode, out, q_len, min_room))
    return rc;
  const long long* rs = reinterpret_cast<const long long*>(row_state);
  const long long* rg = reinterpret_cast<const long long*>(row_geom);
  const long long* rsh = reinterpret_cast<const long long*>(row_share);
  if (layer->d.kv_format == DUO_KV_INT4)
    return launch_decode_ragged_shared_int4(layer, rs, rg, rsh, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len,
                                            scale, workspace, workspace_bytes, (cudaStream_t)stream);
  return launch_decode_ragged_shared(layer, rs, rg, rsh, qkv, qkv_row_stride, cos, sin, rope_mode, out, q_len, scale,
                                     workspace, workspace_bytes, (cudaStream_t)stream);
}

int duo_prefill_ragged(const duo_layer* layer, const int64_t* row_state, const int64_t* row_geom,
                       const int64_t* row_share, const int32_t* lengths, const int64_t* row_room, const void* qkv,
                       int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode, void* out,
                       float scale, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_prefill_ragged";
  (void)workspace;
  (void)workspace_bytes;
  if (!layer || !row_state || !lengths || !row_room) {
    set_error("%s: null argument", who);
    return DUO_EINVAL;
  }
  if (int rc = check_decode_args(who, out != nullptr, qkv, qkv_row_stride, cos, sin, rope_mode)) return rc;
  const duo_layer_desc& d = layer->d;
  if (d.kv_format != DUO_KV_SAME) {
    set_error("%s: 16-bit KV only (prefill the rows of an INT4 cache one at a time)", who);
    return DUO_EINVAL;
  }
  if (d.sink + d.recent > kTcMaxWindow) {
    set_error("%s: sink + recent = %d exceeds %d (prefill such rows one at a time)", who, d.sink + d.recent,
              kTcMaxWindow);
    return DUO_EINVAL;
  }
  if (d.batch > DUO_RAGGED_MAX_BATCH) {
    set_error("%s: batch %d exceeds %d rows", who, d.batch, DUO_RAGGED_MAX_BATCH);
    return DUO_EINVAL;
  }
  if ((layer->pool_tokens != 0) != (row_geom != nullptr) || (row_share && !layer->pool_tokens)) {
    set_error("%s: row_geom (and row_share) go with a pooled layer, and only with one", who);
    return DUO_EINVAL;
  }
  RaggedChunks rc{};
  rc.row_state = reinterpret_cast<const long long*>(row_state);
  rc.row_geom = reinterpret_cast<const long long*>(row_geom);
  rc.row_share = reinterpret_cast<const long long*>(row_share);
  rc.batch = d.batch;
  long long n_tok = 0;
  for (int b = 0; b < d.batch; ++b) {
    const int n = lengths[b];
    if (n < 0) {
      set_error("%s: row %d has a negative chunk length %d", who, b, n);
      return DUO_EINVAL;
    }
    if (d.n_full > 0 && n > row_room[b]) {
      set_error("Trying to put %d KVs into a cache row with room for %lld more (%s, row %d).", n,
                (long long)row_room[b], who, b);
      return DUO_EOVERFLOW;
    }
    if (n > d.stage_cap) {
      set_error("%s: row %d's chunk of %d tokens exceeds the staging capacity %d", who, b, n, d.stage_cap);
      return DUO_EOVERFLOW;
    }
    rc.len[b] = n;
    rc.off[b] = (int)n_tok;
    n_tok += n;
    if (n_tok > INT32_MAX / 2) {
      set_error("%s: %lld packed tokens are too many for one call", who, n_tok);
      return DUO_EINVAL;
    }
  }
  rc.off[d.batch] = (int)n_tok;
  return launch_prefill_ragged(layer, rc, const_cast<void*>(qkv), qkv_row_stride, cos, sin, rope_mode, out, scale,
                               (cudaStream_t)stream);
}

size_t duo_ragged_shared_workspace_bytes(int32_t batch, int32_t n_kv_heads) {
  if (batch < 1 || batch > DUO_RAGGED_MAX_BATCH || n_kv_heads < 1) return 0;
  // one bound for both KV formats: a cache's workspace serves whichever cascade its layers take
  const size_t n = ragged_shared_workspace_bytes(batch, n_kv_heads);
  const size_t n4 = ragged_shared_int4_workspace_bytes(batch, n_kv_heads);
  return n == (size_t)-1 || n4 == (size_t)-1 ? 0 : std::max(n, n4);
}

int duo_ragged_state_advance(int64_t* row_state, int32_t batch, int32_t n, int32_t sink, int32_t recent, void* stream) {
  if (!row_state || batch < 1 || batch > DUO_RAGGED_MAX_BATCH || n < 0 || recent < 1 || sink < 0) {
    set_error("duo_ragged_state_advance: bad argument");
    return DUO_EINVAL;
  }
  return launch_ragged_state_advance(reinterpret_cast<long long*>(row_state), batch, n, sink, recent,
                                     (cudaStream_t)stream);
}

int duo_decode_fused_seq(const duo_layer* layer, const duo_cache_state* st, const void* qkv, int64_t qkv_row_stride,
                         const void* cos, const void* sin, int32_t rope_mode, void* out, float* out_o, float* out_lse,
                         float scale, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_chunk(layer, st, 1, "duo_decode_fused_seq");
  if (!rc)
    rc = check_decode_args("duo_decode_fused_seq", out && out_o && out_lse, qkv, qkv_row_stride, cos, sin, rope_mode);
  if (rc) return rc;
  if (st->seq_world < 2) {
    set_error("duo_decode_fused_seq: the cache state carries no sequence-shard descriptor");
    return DUO_EINVAL;
  }
  if (layer->d.kv_format != DUO_KV_SAME || layer->d.group > 16) {
    set_error("duo_decode_fused_seq: 16-bit caches and group <= 16 only (INT4 caches: duo_decode_fused_seq_int4)");
    return DUO_EINVAL;
  }
  return launch_decode_fused_seq(layer, st, qkv, qkv_row_stride, cos, sin, rope_mode, out, out_o, out_lse, scale, workspace,
                                 workspace_bytes, (cudaStream_t)stream);
}

// The prefix of the forks of a sequence-sharded prompt: a batch-1 handle of the layer's geometry (group16: group <= 16,
// the 16 packed rows of the fork suffix kernel)
static int check_prefix_geometry(const char* who, const duo_layer* layer, const duo_layer* prefix, bool group16) {
  const duo_layer_desc &d = layer->d, &pd = prefix->d;
  if (pd.batch != 1 || d.n_full != pd.n_full || d.n_stream != pd.n_stream || d.group != pd.group ||
      d.head_dim != pd.head_dim || d.dtype != pd.dtype || (group16 && d.group > 16)) {
    set_error("%s: the prefix must be a batch-1 handle of the layer's geometry (n_full, n_stream, group%s, head_dim, "
              "dtype)", who, group16 ? " <= 16" : "");
    return DUO_EINVAL;
  }
  return DUO_OK;
}

// prefix_len of the forks of a sequence-sharded prompt (after shard_desc_ok): whole rounds of world * block positions,
// at most the forks' full_len, and local rows the prefix's retrieval cache holds
static int check_seq_prefix_len(const char* who, const duo_layer* prefix, const duo_cache_state* st, int64_t prefix_len) {
  const duo_layer_desc& pd = prefix->d;
  const long long round = (long long)st->seq_world * st->seq_block, rows = prefix_len / st->seq_world;
  if (prefix_len <= 0 || prefix_len % round != 0 || prefix_len > st->full_len || (pd.n_full > 0 && rows > pd.full_cap)) {
    set_error("%s: prefix_len %lld must be a positive multiple of world * block %lld, at most full_len %lld, and its "
              "%lld local rows at most the prefix's full_cap %lld", who, (long long)prefix_len, round,
              (long long)st->full_len, rows, (long long)pd.full_cap);
    return DUO_EINVAL;
  }
  return DUO_OK;
}

int duo_decode_fused_seq_shared(const duo_layer* layer, const duo_layer* prefix, int64_t prefix_len,
                                const duo_cache_state* st, const void* qkv, int64_t qkv_row_stride, const void* cos,
                                const void* sin, int32_t rope_mode, void* out, float* out_o, float* out_lse, float scale,
                                void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_decode_fused_seq_shared";
  if (!layer || !prefix || !st) {
    set_error("%s: null argument", who);
    return DUO_EINVAL;
  }
  if (int rc = check_decode_args(who, out && out_o && out_lse, qkv, qkv_row_stride, cos, sin, rope_mode)) return rc;
  if (layer->pool_tokens || prefix->pool_tokens || layer->d.kv_format != DUO_KV_SAME ||
      prefix->d.kv_format != DUO_KV_SAME) {
    set_error("%s: 16-bit layers only (not pooled, not INT4)", who);
    return DUO_EINVAL;
  }
  const duo_layer_desc& d = layer->d;
  if (int rc = check_prefix_geometry(who, layer, prefix, true)) return rc;
  if (!shard_desc_ok(st)) {
    set_error("%s: the cache state carries no valid sequence-shard descriptor (rank %d, world %d, block %d)", who,
              st->seq_rank, st->seq_world, st->seq_block);
    return DUO_EINVAL;
  }
  if (int rc = check_seq_prefix_len(who, prefix, st, prefix_len)) return rc;
  // the own slices hold positions [prefix_len, full_len] at the rows of a sharded cache of positions p - prefix_len
  duo_cache_state own = *st;
  own.full_len = st->full_len - prefix_len;
  if (int rc = check_chunk(layer, &own, 1, who)) return rc;
  const size_t need = seq_shared_workspace_bytes(d.batch, d.n_full + d.n_stream);
  if (need == (size_t)-1 || !workspace || workspace_bytes < need) {
    set_error("%s: workspace too small (%zu < %zu)", who, workspace_bytes, need);
    return DUO_EWORKSPACE;
  }
  return launch_decode_fused_seq_shared(layer, prefix, prefix_len, st, qkv, qkv_row_stride, cos, sin, rope_mode, out,
                                        out_o, out_lse, scale, workspace, workspace_bytes, (cudaStream_t)stream);
}

int duo_prefill_seq_shared(const duo_layer* layer, const duo_layer* prefix, int64_t prefix_len, const duo_cache_state* st,
                           const void* q, int64_t q_row_stride, void* out, float* out_o, float* out_lse, int32_t q_len,
                           float scale, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "duo_prefill_seq_shared";
  if (!layer || !prefix || !st || !q || !out || !out_o || !out_lse) {
    set_error("%s: null argument", who);
    return DUO_EINVAL;
  }
  if (layer->pool_tokens || prefix->pool_tokens || layer->d.kv_format != DUO_KV_SAME ||
      prefix->d.kv_format != DUO_KV_SAME) {
    set_error("%s: 16-bit layers only (not pooled, not INT4)", who);
    return DUO_EINVAL;
  }
  const duo_layer_desc& d = layer->d;
  if (int rc = check_prefix_geometry(who, layer, prefix, false)) return rc;
  if (!shard_desc_ok(st) || st->device_state) {
    set_error("%s: the cache state needs a valid sequence-shard descriptor (rank %d, world %d, block %d) and host "
              "occupancy (no device_state)", who, st->seq_rank, st->seq_world, st->seq_block);
    return DUO_EINVAL;
  }
  if (q_len < 1 || (long long)d.group * q_len <= DUO_DECODE_MAX_Q) {
    set_error("%s: chunks of group * q_len > %d rows only (got group %d, q_len %d; one token per fork: "
              "duo_decode_fused_seq_shared)", who, DUO_DECODE_MAX_Q, d.group, q_len);
    return DUO_EINVAL;
  }
  if (int rc = check_seq_prefix_len(who, prefix, st, prefix_len)) return rc;
  const long long rows = prefix_len / st->seq_world;
  if (rows % 8 != 0) {  // the key tile across the donor's rows and the own rows is issued in 8-row pieces
    set_error("%s: the prefix's %lld local rows (prefix_len / world) must be a multiple of 8 (block %d)", who, rows,
              st->seq_block);
    return DUO_EINVAL;
  }
  // the own slices hold positions [prefix_len, full_len + q_len) at the rows of a sharded cache of positions p - prefix_len
  duo_cache_state own = *st;
  own.full_len = st->full_len - prefix_len;
  if (int rc = check_chunk(layer, &own, q_len, who)) return rc;
  if (tc_prefill_supported(layer, st, q_len))
    return launch_attn_tc_seq_shared(layer, prefix, rows, st, q, q_row_stride, out, out_o, out_lse, q_len, scale,
                                     (cudaStream_t)stream);
  return launch_attn_mma_seq_shared(layer, prefix, rows, st, q, q_row_stride, out, out_o, out_lse, q_len, scale,
                                    workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t duo_seq_shared_workspace_bytes(int32_t batch, int32_t n_kv_heads) {
  if (batch < 1 || n_kv_heads < 1) return 0;
  const size_t n = seq_shared_workspace_bytes(batch, n_kv_heads);
  return n == (size_t)-1 ? 0 : n;
}

// test / tuning hook: force the mma.sync kernel family even for shapes the wgmma prefill kernel takes
int duo_attention_mma(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride,
                      void* out, int32_t q_len, float scale, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_chunk(layer, st, q_len, "duo_attention_mma");
  if (rc) return rc;
  if (layer->d.kv_format != DUO_KV_SAME) {
    set_error("duo_attention_mma: 16-bit KV only");
    return DUO_EINVAL;
  }
  return launch_attn_mma(layer, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes,
                         (cudaStream_t)stream);
}

int duo_state_advance(int64_t* device_state, int32_t n, int32_t sink, int32_t recent, void* stream) {
  if (!device_state || n < 0 || recent < 1 || sink < 0) {
    set_error("duo_state_advance: bad argument");
    return DUO_EINVAL;
  }
  return launch_state_advance(reinterpret_cast<long long*>(device_state), n, sink, recent, (cudaStream_t)stream);
}

int duo_state_set(int64_t* device_state, int64_t full_len, int64_t total, int64_t lo, void* stream) {
  if (!device_state || full_len < 0 || total < 0 || lo < 0) {
    set_error("duo_state_set: bad argument");
    return DUO_EINVAL;
  }
  return launch_state_set(reinterpret_cast<long long*>(device_state), full_len, total, lo, (cudaStream_t)stream);
}

int duo_stream_commit(const duo_layer* layer, const duo_cache_state* st, int32_t q_len, void* stream) {
  int rc = check_chunk(layer, st, q_len, "duo_stream_commit");
  if (rc) return rc;
  return launch_stream_commit(layer, st, q_len, (cudaStream_t)stream);
}

int duo_quant_int4(const void* in, int64_t in_row_stride, int64_t rows, void* packed, void* scale, void* zero,
                   void* stream) {
  if (rows < 0 || (rows > 0 && (!in || !packed || !scale || !zero)) || in_row_stride % 4 != 0) {
    set_error("duo_quant_int4: bad argument");
    return DUO_EINVAL;
  }
  return launch_quant_int4(in, in_row_stride, rows, packed, scale, zero, (cudaStream_t)stream);
}

int duo_attention_partial(const duo_layer* layer, int64_t n_keys, const void* q, int64_t q_row_stride, float* out_o,
                          float* out_lse, int32_t q_len, float scale, void* workspace, size_t workspace_bytes,
                          void* stream) {
  if (!layer || !q || !out_o || !out_lse || n_keys < 0 || q_len < 1) {
    set_error("duo_attention_partial: bad argument");
    return DUO_EINVAL;
  }
  if (layer->pool_tokens) {
    set_error("duo_attention_partial: a pooled ragged layer is decoded with duo_decode_ragged_pooled only");
    return DUO_EINVAL;
  }
  if (layer->d.kv_format != DUO_KV_SAME || layer->d.group * q_len > 16) {
    set_error("duo_attention_partial: 16-bit caches and group * q_len <= 16 only (got group %d, q_len %d)",
              layer->d.group, q_len);
    return DUO_EINVAL;
  }
  if (layer->d.n_full > 0 && n_keys > layer->d.full_cap) {
    set_error("duo_attention_partial: n_keys %lld exceeds the cache capacity %lld", (long long)n_keys,
              (long long)layer->d.full_cap);
    return DUO_EOVERFLOW;
  }
  return launch_attn_mma_partial(layer, n_keys, q, q_row_stride, out_o, out_lse, q_len, scale, workspace,
                                 workspace_bytes, (cudaStream_t)stream);
}

int duo_attention_seq(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride, void* out,
                      float* out_o, float* out_lse, int32_t q_len, float scale, void* workspace, size_t workspace_bytes,
                      void* stream) {
  int rc = check_chunk(layer, st, q_len, "duo_attention_seq");
  if (rc) return rc;
  if (!q || !out || !out_o || !out_lse) {
    set_error("duo_attention_seq: null buffer");
    return DUO_EINVAL;
  }
  if (st->seq_world < 2) {
    set_error("duo_attention_seq: the cache state carries no sequence-shard descriptor");
    return DUO_EINVAL;
  }
  if (layer->d.kv_format != DUO_KV_SAME || layer->d.group * q_len > 16) {
    set_error("duo_attention_seq: 16-bit caches and group * q_len <= 16 only (got group %d, q_len %d; INT4 caches: "
              "duo_attention_seq_int4)", layer->d.group, q_len);
    return DUO_EINVAL;
  }
  return launch_attn_mma_seq(layer, st, q, q_row_stride, out, out_o, out_lse, q_len, scale, workspace, workspace_bytes,
                             (cudaStream_t)stream);
}

int duo_prefill_seq(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride, void* out,
                    float* out_o, float* out_lse, int32_t q_len, float scale, void* workspace, size_t workspace_bytes,
                    void* stream) {
  const char* who = "duo_prefill_seq";
  int rc = check_chunk(layer, st, q_len, who);
  if (rc) return rc;
  if (!q || !out || !out_o || !out_lse) {
    set_error("%s: null buffer", who);
    return DUO_EINVAL;
  }
  if (st->seq_world < 2) {
    set_error("%s: the cache state carries no sequence-shard descriptor", who);
    return DUO_EINVAL;
  }
  if (layer->d.kv_format != DUO_KV_SAME) {
    set_error("%s: 16-bit caches only (attend an INT4 slice through its 16-bit image)", who);
    return DUO_EINVAL;
  }
  if (layer->d.group * q_len <= DUO_DECODE_MAX_Q) {
    set_error("%s: chunks of group * q_len > %d rows only (got group %d, q_len %d; decode-sized chunks: "
              "duo_attention_seq)", who, DUO_DECODE_MAX_Q, layer->d.group, q_len);
    return DUO_EINVAL;
  }
  if (st->device_state) {
    set_error("%s: device_state is only supported for chunks of <= %d tokens", who, DUO_DECODE_MAX_Q);
    return DUO_EINVAL;
  }
  if (tc_prefill_supported(layer, st, q_len))
    return launch_attn_tc_seq(layer, st, q, q_row_stride, out, out_o, out_lse, q_len, scale, (cudaStream_t)stream);
  return launch_attn_mma_seq(layer, st, q, q_row_stride, out, out_o, out_lse, q_len, scale, workspace, workspace_bytes,
                             (cudaStream_t)stream);
}

// The INT4 twins of duo_attention_seq / duo_decode_fused_seq (the keys-as-M INT4 decode kernel on the rank's slice).
// Every check runs before any CUDA call.
static int check_seq_int4(const duo_layer* layer, const duo_cache_state* st, int q_len, const char* who,
                          const char* twin) {
  if (st->seq_world < 2) {
    set_error("%s: the cache state carries no sequence-shard descriptor", who);
    return DUO_EINVAL;
  }
  if (layer->d.kv_format != DUO_KV_INT4) {
    set_error("%s: INT4 caches only (16-bit caches are decoded with %s)", who, twin);
    return DUO_EINVAL;
  }
  if (layer->d.group * q_len > DUO_DECODE_MAX_Q_INT4) {
    set_error("%s: group * q_len <= %d only (got group %d, q_len %d)", who, DUO_DECODE_MAX_Q_INT4, layer->d.group,
              q_len);
    return DUO_EINVAL;
  }
  return DUO_OK;
}

int duo_attention_seq_int4(const duo_layer* layer, const duo_cache_state* st, const void* q, int64_t q_row_stride,
                           void* out, float* out_o, float* out_lse, int32_t q_len, float scale, void* workspace,
                           size_t workspace_bytes, void* stream) {
  const char* who = "duo_attention_seq_int4";
  int rc = check_chunk(layer, st, q_len, who);
  if (rc) return rc;
  if (!q || !out || !out_o || !out_lse) {
    set_error("%s: null buffer", who);
    return DUO_EINVAL;
  }
  if (q_row_stride % 8 != 0 || (reinterpret_cast<uintptr_t>(q) & 15)) {  // the kernel loads q 16 bytes at a time
    set_error("%s: q rows must be 16-byte aligned (row stride a multiple of 8 elements)", who);
    return DUO_EINVAL;
  }
  if (int rc2 = check_seq_int4(layer, st, q_len, who, "duo_attention_seq")) return rc2;
  return launch_attn_int4_seq(layer, st, q, q_row_stride, out, out_o, out_lse, q_len, scale, workspace, workspace_bytes,
                              (cudaStream_t)stream);
}

int duo_decode_fused_seq_int4(const duo_layer* layer, const duo_cache_state* st, const void* qkv,
                              int64_t qkv_row_stride, const void* cos, const void* sin, int32_t rope_mode, void* out,
                              float* out_o, float* out_lse, float scale, void* workspace, size_t workspace_bytes,
                              void* stream) {
  const char* who = "duo_decode_fused_seq_int4";
  int rc = check_chunk(layer, st, 1, who);
  if (!rc) rc = check_decode_args(who, out && out_o && out_lse, qkv, qkv_row_stride, cos, sin, rope_mode);
  if (!rc) rc = check_seq_int4(layer, st, 1, who, "duo_decode_fused_seq");
  if (rc) return rc;
  return launch_decode_fused_seq_int4(layer, st, qkv, qkv_row_stride, cos, sin, rope_mode, out, out_o, out_lse, scale,
                                      workspace, workspace_bytes, (cudaStream_t)stream);
}

int duo_merge_partials(const float* o_parts, const float* lse_parts, int32_t n_parts, int64_t tokens,
                       int32_t heads_total, int32_t heads_used, void* out, int32_t dtype, void* stream) {
  if (n_parts < 1 || tokens < 0 || heads_total < 1 || heads_used < 0 || heads_used > heads_total ||
      (tokens > 0 && heads_used > 0 && (!o_parts || !lse_parts || !out)) ||
      (dtype != DUO_DT_BF16 && dtype != DUO_DT_FP16)) {
    set_error("duo_merge_partials: bad argument");
    return DUO_EINVAL;
  }
  return launch_merge_partials(o_parts, lse_parts, n_parts, tokens, heads_total, heads_used, out, dtype,
                               (cudaStream_t)stream);
}

int duo_add_rmsnorm(const void* x, const void* residual, const void* weight, void* out_norm, void* out_res, int64_t rows,
                    int32_t hidden, float eps, int32_t dtype, void* stream) {
  if (rows < 0 || hidden < 8 || hidden % 8 != 0 || hidden > 16384 || (rows > 0 && (!x || !weight || !out_norm)) ||
      (dtype != DUO_DT_BF16 && dtype != DUO_DT_FP16)) {
    set_error("duo_add_rmsnorm: bad argument");
    return DUO_EINVAL;
  }
  return launch_add_rmsnorm(x, residual, weight, out_norm, out_res, rows, hidden, eps, dtype, (cudaStream_t)stream);
}

int duo_silu_mul(const void* gate_up, void* out, int64_t rows, int32_t inter, int32_t dtype, void* stream) {
  if (rows < 0 || inter < 8 || inter % 8 != 0 || (rows > 0 && (!gate_up || !out)) ||
      (dtype != DUO_DT_BF16 && dtype != DUO_DT_FP16)) {
    set_error("duo_silu_mul: bad argument");
    return DUO_EINVAL;
  }
  return launch_silu_mul(gate_up, out, rows, inter, dtype, (cudaStream_t)stream);
}

int duo_dequant_int4(const void* packed, const void* scale, const void* zero, int64_t rows, void* out, void* stream) {
  if (rows < 0 || (rows > 0 && (!packed || !scale || !zero || !out))) {
    set_error("duo_dequant_int4: bad argument");
    return DUO_EINVAL;
  }
  return launch_dequant_int4(packed, scale, zero, rows, out, (cudaStream_t)stream);
}

int duo_dequant_int4_bf16(const void* packed, const void* scale, const void* zero, int64_t rows, void* out,
                          void* stream) {
  if (rows < 0 || (rows > 0 && (!packed || !scale || !zero || !out))) {
    set_error("duo_dequant_int4_bf16: bad argument");
    return DUO_EINVAL;
  }
  return launch_dequant_int4_bf16(packed, scale, zero, rows, out, (cudaStream_t)stream);
}

}  // extern "C"
