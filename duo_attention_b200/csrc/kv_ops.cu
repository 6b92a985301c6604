// KV-side kernels of the hot path: RoPE + cache append (+ INT4 quantise), streaming ring commit,
// stand-alone INT4 quantise / dequantise.  All HBM-bound byte work: one warp per 128-element row,
// 8-byte vector loads (a full row = one 256 B coalesced request), warp-shuffle reductions.
//
// Reference semantics restated here:
//   RoPE (HF op order)       duo_attn/patch/llama.py:177-184 -> transformers apply_rotary_pos_emb
//   RoPE (fp32, flashinfer)  duo_attn/patch/flashinfer_utils.py:29-59
//   append                   duo_attn/patch/static_kv_cache.py:109-125, 252-263
//   ring commit              duo_attn/patch/static_kv_cache.py:127-167 / llama.py:273-290
//   INT4 K1 / K2             demo/quantize_int4.cu:73-144 / :9-42 (K2's __hadd(__hmul()) is contracted by nvcc
//                            into one HFMA2 in the reference build — verified in its SASS — so K2 == fma)
// K1 runs on the fp32 value of each (rotated) fp16 or bf16 row; rows of a bf16 layer must lie within fp16 range,
// since scale / zero are stored as fp16.
#include "duo_common.cuh"

namespace duo {

int stage_offset(const duo_layer_desc& d);  // api.cu

struct RopeAppendParams {
  void* qkv;
  long long row_stride;  // elements between consecutive tokens
  const void* cos;
  const void* sin;
  int rope_mode;
  int q_len, batch, n_q, n_kv, n_full, n_stream;
  int W, ring_slots;  // first staging slot, staging slot + stage_cap
  int skip_q;
  long long full_cap, full_len;
  const long long* dstate;
  int kv_int4;
  int seq_rank, seq_world, seq_block;  // sequence-sharded retrieval caches (duo_cache_state): append owned positions only
  void *full_k, *full_v, *ring_k, *ring_v;
  __half *fks, *fkz, *fvs, *fvz, *rks, *rkz, *rvs, *rvz;
};

// RAGGED (duo_prefill_ragged): the rows are the packed chunks of RaggedChunks (p.q_len = their total T, p.batch = 1):
// packed token o_b + t is token t of row b, rotated with row o_b + t of the packed cos / sin tables; its retrieval K/V go
// to row full_len_b + t of row b's cache (a sharer's: own region row full_len_b - P_b + t), its streaming K/V to row b's
// staging slot W + t.  (The RaggedChunks parameter follows p, so p's offsets are those of every instantiation.)
template <typename T, bool RAGGED = false>
__global__ void __launch_bounds__(256) rope_append_kernel(const RopeAppendParams p, const __grid_constant__ RaggedChunks rc) {
  const int lane = threadIdx.x & 31;
  const int slots = p.n_q + 2 * p.n_kv;
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total_rows = (long long)p.batch * p.q_len * slots;
  if (wid >= total_rows) return;
  const int slot = (int)(wid % slots);
  const long long bt = wid / slots;
  int t = (int)(bt % p.q_len);
  int b = (int)(bt / p.q_len);
  if constexpr (RAGGED) {
    b = ragged_chunk_row(rc, bt);
    t = (int)(bt - rc.off[b]);
  }

  T* row = reinterpret_cast<T*>(p.qkv) + (bt * p.row_stride) + (long long)slot * kHeadDim;
  Vec4<T> xv = *reinterpret_cast<const Vec4<T>*>(row + lane * 4);
  const bool is_q = slot < p.n_q;
  const bool is_k = !is_q && slot < p.n_q + p.n_kv;
  const bool is_v = !is_q && !is_k;

  float xo[4];  // values as they will be stored (already rounded to T)
  if (!is_v && p.rope_mode != DUO_ROPE_NONE) rope_row4<T>(xv, lane, RAGGED ? (int)bt : t, p.cos, p.sin, p.rope_mode);
#pragma unroll
  for (int i = 0; i < 4; ++i) xo[i] = RopeCvt<T>::to_f(xv.v[i]);

  if (is_q) {
    if (p.rope_mode != DUO_ROPE_NONE && !p.skip_q) *reinterpret_cast<Vec4<T>*>(row + lane * 4) = xv;
    return;
  }
  const int h = is_k ? slot - p.n_q : slot - p.n_q - p.n_kv;
  const bool full = h < p.n_full;
  long long dst_row;  // row index inside the destination tensor
  const long long full_len = p.dstate ? p.dstate[0] : p.full_len;
  if constexpr (RAGGED) {
    if (full) {
      int donor;
      const long long row = rc.row_state[4 * b] - ragged_chunk_share(rc, b, donor) + t;
      dst_row = rc.row_geom ? ragged_pool_row(rc, b, p.n_full, h, row) : ((long long)b * p.n_full + h) * p.full_cap + row;
    } else {
      dst_row = ((long long)b * p.n_stream + (h - p.n_full)) * p.ring_slots + p.W + t;
    }
  } else if (full) {
    long long row = full_len + t;
    if (p.seq_world > 1) {  // block-cyclic slice: position -> (owner, local row); other ranks' positions are skipped
      const long long blk = row / p.seq_block;
      if ((int)(blk % p.seq_world) != p.seq_rank) return;
      row = (blk / p.seq_world) * p.seq_block + row % p.seq_block;
    }
    dst_row = ((long long)b * p.n_full + h) * p.full_cap + row;
  } else
    dst_row = ((long long)b * p.n_stream + (h - p.n_full)) * p.ring_slots + p.W + t;
  void* base = full ? (is_k ? p.full_k : p.full_v) : (is_k ? p.ring_k : p.ring_v);
  if (!p.kv_int4) {
    *reinterpret_cast<Vec4<T>*>(reinterpret_cast<T*>(base) + dst_row * kHeadDim + lane * 4) = xv;
  } else {
    __half* sc = full ? (is_k ? p.fks : p.fvs) : (is_k ? p.rks : p.rvs);
    __half* zp = full ? (is_k ? p.fkz : p.fvz) : (is_k ? p.rkz : p.rvz);
    quant_row_int4(xo, lane, reinterpret_cast<uint8_t*>(base) + dst_row * (kHeadDim / 2), sc + dst_row, zp + dst_row);
  }
}

int launch_rope_append(const duo_layer* L, const duo_cache_state* st, void* qkv, long long row_stride, const void* cos,
                       const void* sin, int rope_mode, int q_len, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  RopeAppendParams p{};
  p.qkv = qkv;
  p.row_stride = row_stride;
  p.cos = cos;
  p.sin = sin;
  p.rope_mode = rope_mode & 0xff;
  p.skip_q = (rope_mode & DUO_ROPE_SKIP_Q) ? 1 : 0;
  p.q_len = q_len;
  p.batch = d.batch;
  p.n_kv = d.n_full + d.n_stream;
  p.n_q = p.n_kv * d.group;
  p.n_full = d.n_full;
  p.n_stream = d.n_stream;
  p.W = stage_offset(d);
  p.ring_slots = p.W + d.stage_cap;
  p.full_cap = d.full_cap;
  p.full_len = st->full_len;
  p.dstate = reinterpret_cast<const long long*>(st->device_state);
  p.kv_int4 = d.kv_format == DUO_KV_INT4;
  p.seq_rank = st->seq_rank;
  p.seq_world = st->seq_world;
  p.seq_block = st->seq_block;
  p.full_k = d.full_k;
  p.full_v = d.full_v;
  p.ring_k = d.ring_k;
  p.ring_v = d.ring_v;
  p.fks = (__half*)d.full_k_scale;
  p.fkz = (__half*)d.full_k_zero;
  p.fvs = (__half*)d.full_v_scale;
  p.fvz = (__half*)d.full_v_zero;
  p.rks = (__half*)d.ring_k_scale;
  p.rkz = (__half*)d.ring_k_zero;
  p.rvs = (__half*)d.ring_v_scale;
  p.rvz = (__half*)d.ring_v_zero;
  const long long rows = (long long)d.batch * q_len * (p.n_q + 2 * p.n_kv);
  const int wpb = 8;
  const long long blocks = (rows + wpb - 1) / wpb;
  if (blocks == 0) return DUO_OK;
  if (d.dtype == DUO_DT_BF16)
    rope_append_kernel<__nv_bfloat16><<<(unsigned)blocks, wpb * 32, 0, stream>>>(p, RaggedChunks{});
  else
    rope_append_kernel<__half><<<(unsigned)blocks, wpb * 32, 0, stream>>>(p, RaggedChunks{});
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

// The append of a batched ragged prefill (16-bit layers): every row's chunk in one launch, see rope_append_kernel.
int launch_rope_append_ragged(const duo_layer* L, const RaggedChunks& rc, void* qkv, long long row_stride,
                              const void* cos, const void* sin, int rope_mode, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  RopeAppendParams p{};
  p.qkv = qkv;
  p.row_stride = row_stride;
  p.cos = cos;
  p.sin = sin;
  p.rope_mode = rope_mode & 0xff;
  p.q_len = rc.off[rc.batch];
  p.batch = 1;
  p.n_kv = d.n_full + d.n_stream;
  p.n_q = p.n_kv * d.group;
  p.n_full = d.n_full;
  p.n_stream = d.n_stream;
  p.W = stage_offset(d);
  p.ring_slots = p.W + d.stage_cap;
  p.full_cap = d.full_cap;
  p.full_k = d.full_k;
  p.full_v = d.full_v;
  p.ring_k = d.ring_k;
  p.ring_v = d.ring_v;
  const long long rows = (long long)p.q_len * (p.n_q + 2 * p.n_kv);
  const int wpb = 8;
  const long long blocks = (rows + wpb - 1) / wpb;
  if (blocks == 0) return DUO_OK;
  if (d.dtype == DUO_DT_BF16)
    rope_append_kernel<__nv_bfloat16, true><<<(unsigned)blocks, wpb * 32, 0, stream>>>(p, rc);
  else
    rope_append_kernel<__half, true><<<(unsigned)blocks, wpb * 32, 0, stream>>>(p, rc);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

// ---------------------------------------------------------------------------------------------
// ring commit: staged chunk rows -> sink / ring slots
// ---------------------------------------------------------------------------------------------
struct CommitParams {
  uint8_t *ring_k, *ring_v;
  __half *rks, *rkz, *rvs, *rvz;
  int row_bytes;  // 256 (16-bit) or 64 (int4)
  int kv_int4;
  int batch, n_stream, ring_slots, W /* first staging slot */, sink, recent, q_len;
  long long total;
  const long long* dstate;  // when set: total is read from device memory and all q_len rows are candidates
  int n_cand;      // candidate chunk rows per head: sinks first, then the tail
  int n_sink_new;  // chunk rows [0, n_sink_new) land in sink slots
  int tail_start;  // chunk rows [tail_start, q_len) land in the ring
};

// RAGGED (duo_prefill_ragged): p.n_cand = the packed tokens T, p.batch = 1; packed token o_b + i is chunk row i of row b,
// committed against row b's total from row_state as the device-state path does, into row b's ring.
template <bool RAGGED = false>
__global__ void __launch_bounds__(256) stream_commit_kernel(const CommitParams p, const __grid_constant__ RaggedChunks rc) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total_rows = (long long)p.batch * p.n_stream * p.n_cand * 2;
  if (wid >= total_rows) return;
  const int kv = (int)(wid & 1);
  long long x = wid >> 1;
  const int c = (int)(x % p.n_cand);
  long long bh = x / p.n_cand;
  int i;
  long long total = p.total;
  if constexpr (RAGGED) {
    const int b = ragged_chunk_row(rc, c);
    const int len = rc.len[b];
    i = c - rc.off[b];
    total = rc.row_state[4 * b + 1];
    if (!(total + i < p.sink || i >= len - p.recent)) return;
    bh += (long long)b * p.n_stream;  // bh = the streaming head here (p.batch = 1)
  } else if (p.dstate) {
    total = p.dstate[1];
    i = c;  // every chunk row is a candidate; keep sinks and the last `recent` rows
    if (!(total + i < p.sink || i >= p.q_len - p.recent)) return;
  } else if (c < p.n_sink_new) {
    i = c;
  } else {
    i = p.tail_start + (c - p.n_sink_new);
  }
  if (!RAGGED && i >= p.q_len) return;
  const long long pos = total + i;
  int slot;
  if (pos < p.sink)
    slot = (int)pos;
  else
    slot = p.sink + (int)((pos - p.sink) % p.recent);
  const long long src = bh * p.ring_slots + p.W + i;
  const long long dst = bh * p.ring_slots + slot;
  uint8_t* base = kv ? p.ring_v : p.ring_k;
  if (p.row_bytes == 256) {
    const uint2 v = *reinterpret_cast<const uint2*>(base + src * 256 + lane * 8);
    *reinterpret_cast<uint2*>(base + dst * 256 + lane * 8) = v;
  } else {
    const uint16_t v = *reinterpret_cast<const uint16_t*>(base + src * 64 + lane * 2);
    *reinterpret_cast<uint16_t*>(base + dst * 64 + lane * 2) = v;
    if (lane == 0) {
      __half* sc = kv ? p.rvs : p.rks;
      __half* zp = kv ? p.rvz : p.rkz;
      sc[dst] = sc[src];
      zp[dst] = zp[src];
    }
  }
}

int launch_stream_commit(const duo_layer* L, const duo_cache_state* st, int q_len, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  if (d.n_stream == 0 || q_len == 0) return DUO_OK;
  CommitParams p{};
  p.ring_k = (uint8_t*)d.ring_k;
  p.ring_v = (uint8_t*)d.ring_v;
  p.rks = (__half*)d.ring_k_scale;
  p.rkz = (__half*)d.ring_k_zero;
  p.rvs = (__half*)d.ring_v_scale;
  p.rvz = (__half*)d.ring_v_zero;
  p.kv_int4 = d.kv_format == DUO_KV_INT4;
  p.row_bytes = p.kv_int4 ? 64 : 256;
  p.batch = d.batch;
  p.n_stream = d.n_stream;
  p.W = stage_offset(d);
  p.ring_slots = p.W + d.stage_cap;
  p.sink = d.sink;
  p.recent = d.recent;
  p.q_len = q_len;
  p.total = st->total;
  // chunk rows i with position total+i < sink are sinks; of the rest only the last `recent` survive
  long long n_sink_new = d.sink - st->total;
  if (n_sink_new < 0) n_sink_new = 0;
  if (n_sink_new > q_len) n_sink_new = q_len;
  int tail_start = q_len - d.recent;
  if (tail_start < (int)n_sink_new) tail_start = (int)n_sink_new;
  p.n_sink_new = (int)n_sink_new;
  p.tail_start = tail_start;
  p.n_cand = (int)n_sink_new + (q_len - tail_start);
  p.dstate = reinterpret_cast<const long long*>(st->device_state);
  if (p.dstate) p.n_cand = q_len;
  if (p.n_cand <= 0) return DUO_OK;
  const long long rows = (long long)d.batch * d.n_stream * p.n_cand * 2;
  const long long blocks = (rows + 7) / 8;
  stream_commit_kernel<<<(unsigned)blocks, 256, 0, stream>>>(p, RaggedChunks{});
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

// The commit of a batched ragged prefill (16-bit layers): every row's staged chunk in one launch.
int launch_stream_commit_ragged(const duo_layer* L, const RaggedChunks& rc, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  const int n_tok = rc.off[rc.batch];
  if (d.n_stream == 0 || n_tok == 0) return DUO_OK;
  CommitParams p{};
  p.ring_k = (uint8_t*)d.ring_k;
  p.ring_v = (uint8_t*)d.ring_v;
  p.row_bytes = 256;
  p.batch = 1;
  p.n_stream = d.n_stream;
  p.W = stage_offset(d);
  p.ring_slots = p.W + d.stage_cap;
  p.sink = d.sink;
  p.recent = d.recent;
  p.q_len = n_tok;
  p.n_cand = n_tok;
  const long long rows = (long long)d.n_stream * n_tok * 2;
  const long long blocks = (rows + 7) / 8;
  stream_commit_kernel<true><<<(unsigned)blocks, 256, 0, stream>>>(p, rc);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

// ---------------------------------------------------------------------------------------------
// stand-alone INT4 quantise / dequantise (K1 / K2)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) quant_int4_kernel(const __half* in, long long in_row_stride, long long rows,
                                                         uint8_t* packed, __half* scale, __half* zero) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const Vec4<__half> xv = *reinterpret_cast<const Vec4<__half>*>(in + r * in_row_stride + lane * 4);
  float x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = __half2float(xv.v[i]);
  quant_row_int4(x, lane, packed + r * 64, scale + r, zero + r);
}

__global__ void __launch_bounds__(256) dequant_int4_kernel(const uint8_t* packed, const __half* scale,
                                                           const __half* zero, long long rows, __half* out) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const uint16_t two = *reinterpret_cast<const uint16_t*>(packed + r * 64 + lane * 2);
  const __half s = scale[r], z = zero[r];
  const uint32_t b0 = two & 0xff, b1 = two >> 8;
  const uint32_t q[4] = {b0 >> 4, b0 & 0xf, b1 >> 4, b1 & 0xf};
  Vec4<__half> o;
#pragma unroll
  for (int i = 0; i < 4; ++i) o.v[i] = __hfma(__float2half((float)q[i]), s, z);  // as-built reference: HFMA2, one rounding
  *reinterpret_cast<Vec4<__half>*>(out + r * 128 + lane * 4) = o;
}

// bf16 image of an INT4 row for a bf16 layer: bf16_rn(fmaf(code, scale, zero)) with fp32 scale / zero (exact widenings
// of the stored fp16 values).  A different rounding from K2 (which rounds the same fma to fp16), not a re-rounding of it.
__global__ void __launch_bounds__(256) dequant_int4_bf16_kernel(const uint8_t* packed, const __half* scale,
                                                                const __half* zero, long long rows, __nv_bfloat16* out) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const uint16_t two = *reinterpret_cast<const uint16_t*>(packed + r * 64 + lane * 2);
  const float s = __half2float(scale[r]), z = __half2float(zero[r]);
  const uint32_t b0 = two & 0xff, b1 = two >> 8;
  const uint32_t q[4] = {b0 >> 4, b0 & 0xf, b1 >> 4, b1 & 0xf};
  Vec4<__nv_bfloat16> o;
#pragma unroll
  for (int i = 0; i < 4; ++i) o.v[i] = __float2bfloat16_rn(__fmaf_rn((float)q[i], s, z));
  *reinterpret_cast<Vec4<__nv_bfloat16>*>(out + r * 128 + lane * 4) = o;
}

__global__ void state_advance_kernel(long long* st, int n, int sink, int recent) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const long long total = st[1] + n;
    st[0] += n;
    st[1] = total;
    long long lo = st[2];
    if (total - recent > lo) lo = total - recent;
    if (lo < sink) lo = sink;
    st[2] = lo;
  }
}

__global__ void state_set_kernel(long long* st, long long full_len, long long total, long long lo) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    st[0] = full_len;
    st[1] = total;
    st[2] = lo;
  }
}

int launch_state_set(long long* st, long long full_len, long long total, long long lo, cudaStream_t stream) {
  state_set_kernel<<<1, 32, 0, stream>>>(st, full_len, total, lo);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

int launch_state_advance(long long* st, int n, int sink, int recent, cudaStream_t stream) {
  state_advance_kernel<<<1, 32, 0, stream>>>(st, n, sink, recent);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

// row_state [batch][4] = {full_len, total, lo, flags}: every active row advances as state_advance_kernel does, an idle
// one (ragged_idle) keeps its state
__global__ void ragged_state_advance_kernel(long long* st, int batch, int n, int sink, int recent) {
  const int r = threadIdx.x;
  if (blockIdx.x == 0 && r < batch && !ragged_idle(st, r)) {
    long long* s = st + 4 * r;
    const long long total = s[1] + n;
    s[0] += n;
    s[1] = total;
    long long lo = s[2];
    if (total - recent > lo) lo = total - recent;
    if (lo < sink) lo = sink;
    s[2] = lo;
  }
}

int launch_ragged_state_advance(long long* st, int batch, int n, int sink, int recent, cudaStream_t stream) {
  ragged_state_advance_kernel<<<1, 64, 0, stream>>>(st, batch, n, sink, recent);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

int launch_quant_int4(const void* in, long long in_row_stride, long long rows, void* packed, void* scale, void* zero,
                      cudaStream_t stream) {
  if (rows == 0) return DUO_OK;
  const long long blocks = (rows + 7) / 8;
  quant_int4_kernel<<<(unsigned)blocks, 256, 0, stream>>>((const __half*)in, in_row_stride, rows, (uint8_t*)packed,
                                                          (__half*)scale, (__half*)zero);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

int launch_dequant_int4(const void* packed, const void* scale, const void* zero, long long rows, void* out,
                        cudaStream_t stream) {
  if (rows == 0) return DUO_OK;
  const long long blocks = (rows + 7) / 8;
  dequant_int4_kernel<<<(unsigned)blocks, 256, 0, stream>>>((const uint8_t*)packed, (const __half*)scale,
                                                            (const __half*)zero, rows, (__half*)out);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

int launch_dequant_int4_bf16(const void* packed, const void* scale, const void* zero, long long rows, void* out,
                             cudaStream_t stream) {
  if (rows == 0) return DUO_OK;
  const long long blocks = (rows + 7) / 8;
  dequant_int4_bf16_kernel<<<(unsigned)blocks, 256, 0, stream>>>((const uint8_t*)packed, (const __half*)scale,
                                                                 (const __half*)zero, rows, (__nv_bfloat16*)out);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

}  // namespace duo
