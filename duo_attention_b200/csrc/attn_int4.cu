// Mixed-head attention over an INT4 KV cache with the dequantisation FOLDED INTO THE K/V LOAD.
//
// The reference dequantises the whole cache to an fp16 scratch buffer on every layer of every step
// (demo/int4_kv.py:373-436: an O(ctx) write + re-read) and then calls flash_attn_func on it
// (demo/w8a8kv4_llama.py:239-274).  Here the packed nibbles go HBM -> smem -> registers -> tensor cores and the
// per-row scale / zero-point are applied algebraically on the 16 x keys logits / 16 x 128 outputs instead of on
// the keys x 128 elements:
//
//   S[r,j] = s_j * (Q_r . c_j) + z_j * sum(Q_r)                 c_j = 4-bit codes of key j
//   O[r,:] = sum_j (p_rj s_j) c_j  +  sum_j p_rj z_j
//
// nibble -> fp16 costs 5 ALU ops per 8 nibbles: (w & 0x000f000f) | 0x64006400 is the half2 (1024+c_a, 1024+c_b)
// and (w & 0x00f000f0) | 0x64006400 is (1024+16 c_a', 1024+16 c_b'); the +1024 offsets and the x16 are removed
// algebraically (Q pre-scaled by 1/16 on the "high nibble" slots, offsets subtracted per row), so no per-element
// subtract / multiply is ever issued.  Because a dot product is permutation invariant the head_dim order inside
// a k16 step is chosen to match what these masks produce; V codes are transposed for the PV product by
// ldmatrix.trans on 16-bit units (4 codes of one key), which lands the same head_dim column of two adjacent
// keys in one register - exactly the (0x000f000f) pattern again.
//
// Tiles (64 keys: 4 KB K + 4 KB V + 4 x 128 B scale/zero = 8.5 KB instead of 32 KB) are fetched with 16 B
// cp.async (zero-fill beyond the valid rows) into a 4-stage ring.  Same work decomposition, masks, split-KV merge
// and variants as attn_mma.cu.
//
// Activations are fp16 (the reference's INT4 demo runs in fp16) or bf16 (T = __nv_bfloat16).  The inner loop is fp16
// in both cases: the nibble -> fp16 trick and the 1/16 pre-scale of the high-nibble slots need fp16's 10-bit mantissa
// (bf16's 7 bits cannot hold 1024 + 16 c), and the fp16 scale / zero of the format already require K and V to lie in
// fp16 range.  A bf16 kernel loads q (and, fused, the new K / V rows) as bf16, applies RoPE in bf16 with the same
// device functions as the 16-bit path, converts q to fp16 (round to nearest) where the fragments are built, and stores
// its outputs as bf16; P' = p s_v stays rounded to fp16.  Hence the one extra limit of the bf16 path: q must lie within
// fp16's finite range (|q| <= 65504); elements below 2^-14 in magnitude become fp16 subnormals (absolute error
// <= 2^-25).  The new K / V rows are quantised (K1) from the fp32 value of the rotated bf16 row, exactly as
// rope_append_kernel<bf16> does.
//
// The decode kernel (duo_attn_int4_dec8_kernel, group x q_len <= 8) swaps the operand roles (keys are the MMA M) and, as
// duo_decode_fused, is the whole decode step of a layer in one launch: q RoPE in registers, RoPE + K1 quantisation +
// append of the new K / V by the CTA that reads those rows, ring commit by the streaming-head CTA.
#include <cstdlib>
#include <type_traits>

#include "duo_common.cuh"

namespace duo {

// keys per pipeline stage: 128 for the decode variant (4 key-warps x 32 keys: halves the per-tile fixed cost of
// the ALU-bound loop), 64 for the 64-row chunk variant
template <int KEY_WARPS>
struct I4Cfg {
  static constexpr int TILE = KEY_WARPS == 4 ? 128 : 64;
  static constexpr int STAGES = KEY_WARPS == 4 ? 3 : 4;
  static constexpr int PACK_BYTES = TILE * 64;                  // one packed K or V tile
  static constexpr int STAGE_BYTES = 2 * PACK_BYTES + 4 * TILE * 2;  // + k_scale, k_zero, v_scale, v_zero
};
constexpr int I4_THREADS = 128;
constexpr int I4_MERGE_BYTES = 96 * 1024;  // smem the split-KV merge needs (see attn_mma.cu); >= every pipeline
constexpr int I4_SMEM_BYTES = I4_MERGE_BYTES + 128;

struct I4Params {
  const void* q;
  void* out;
  long long q_tok_stride, q_batch_stride, out_batch_stride;
  int q_len, n_q_heads, group, n_full, n_stream, batch;
  int sink, recent, W, stage_off;
  long long full_len, total, lo;
  const long long* dstate;
  long long full_cap, ring_slots;
  float scale_log2;
  int splits_full, keys_per_split, n_rb, cache_scan;
  SplitWs ws;  // split-KV partials + arrival counters (duo_common.cuh)
  const uint8_t *full_k, *full_v, *ring_k, *ring_v;
  const __half *fks, *fkz, *fvs, *fvz, *rks, *rkz, *rvs, *rvz;
  // FUSED decode step (duo_decode_fused on an INT4 cache, duo_attn_int4_dec8_kernel<true>): `q` points at the RAW fused
  // qkv rows; the kernel rotates q in registers, and the CTA that owns the end of a head's key range rotates the new
  // tokens' K, quantises K / V (K1) into the cache rows the loop then reads, and commits the streaming ring at the end.
  const void *cos, *sin;
  int rope_mode;
  long long k_off, v_off;  // element offsets of the k / v sections inside a qkv row
  // RAGGED decode (duo_decode_ragged_int4, duo_attn_int4_dec8_kernel<true, T, true>): `dstate` is the [batch][4]
  // row_state array, every batch row has its own occupancy, and the retrieval CTAs of a kv head are rg_slots grid
  // slots shared by all rows (see AttnParams in attn_mma.cu).
  int rg_slots;
  int rg_want;  // split budget per (row, retrieval head) at equal lengths: the `want` of launch_i4_dec8
  // POOLED ragged decode (duo_decode_ragged_pooled): full_k / full_v and their scale / zero rows are pools of
  // pool_tokens * n_full rows; row_geom [batch][2] = {first_b, cap_b} places row b's [n_full][cap_b] region at pool
  // row first_b * n_full (see AttnParams in attn_mma.cu).
  const long long* row_geom;
  // SEQUENCE-SHARDED decode (duo_attention_seq_int4 / duo_decode_fused_seq_int4, duo_attn_int4_dec8_kernel<.., SEQ>):
  // `full_len` counts GLOBAL tokens and the retrieval cache holds the block-cyclic slice of rank seq_rank; retrieval
  // heads write the fp32 normalised O and log2-domain log-sum-exp of that slice to part_o / part_lse instead of `out`
  // (the contract of AttnParams in attn_mma.cu), streaming heads run as unsharded.
  float* part_o;
  float* part_lse;
  int seq_rank, seq_world, seq_block;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// (w & mask) | 0x64006400 as ONE LOP3 (the C expression compiles to two, both with immediate operands):
//   lop1_lo: half2(1024 + nib[bits 0-3], 1024 + nib[bits 16-19])
//   lop1_hi: half2(1024 + 16 nib[bits 4-7], 1024 + 16 nib[bits 20-23])
__device__ __forceinline__ uint32_t lop3_and_or(uint32_t w, uint32_t mask, uint32_t magic) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(w), "r"(mask), "r"(magic));
  return d;
}
__device__ __forceinline__ uint32_t lop1_lo(uint32_t w) { return lop3_and_or(w, 0x000f000fu, 0x64006400u); }
__device__ __forceinline__ uint32_t lop1_hi(uint32_t w) { return lop3_and_or(w, 0x00f000f0u, 0x64006400u); }

// activation element -> the fp16 the inner loop works in (identity for fp16 activations)
__device__ __forceinline__ __half to_half(__half v) { return v; }
__device__ __forceinline__ __half to_half(__nv_bfloat16 v) { return __float2half_rn(__bfloat162float(v)); }

template <int KEY_WARPS, typename T>
__global__ void __launch_bounds__(I4_THREADS, 2) duo_attn_int4_kernel(const I4Params pin) {
  I4Params p = pin;
  if (pin.dstate) {  // occupancy lives in device memory (CUDA-graph replay)
    p.full_len = pin.dstate[0];
    p.total = pin.dstate[1];
    p.lo = pin.dstate[2];
    const long long nk = p.full_len + p.q_len;
    p.keys_per_split = (int)split_keys(nk, p.splits_full, I4Cfg<KEY_WARPS>::TILE);
    p.cache_scan = (int)(p.total < p.W ? p.total : p.W);
  }
  constexpr int ROW_WARPS = 4 / KEY_WARPS;
  constexpr int ROWS = 16 * ROW_WARPS;
  constexpr int I4_TILE = I4Cfg<KEY_WARPS>::TILE;
  constexpr int I4_STAGES = I4Cfg<KEY_WARPS>::STAGES;
  constexpr int I4_PACK_BYTES = I4Cfg<KEY_WARPS>::PACK_BYTES;
  constexpr int I4_STAGE_BYTES = I4Cfg<KEY_WARPS>::STAGE_BYTES;
  constexpr int KPW = I4_TILE / KEY_WARPS;
  constexpr int NT = KPW / 8;
  using Op = MmaOp<__half>;

  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  __shared__ int s_is_last;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.y;

  // ---- work item (same enumeration as attn_mma.cu) ----------------------------------------------
  const int n_full_items = p.n_full * p.n_rb * p.splits_full;
  int kvh, rb, split;
  bool is_full;
  if ((int)blockIdx.x < n_full_items) {
    is_full = true;
    int x = blockIdx.x;
    split = x % p.splits_full;
    x /= p.splits_full;
    rb = p.n_rb - 1 - (x % p.n_rb);
    kvh = x / p.n_rb;
  } else {
    is_full = false;
    int x = blockIdx.x - n_full_items;
    rb = p.n_rb - 1 - (x % p.n_rb);
    kvh = p.n_full + x / p.n_rb;
    split = 0;
  }
  const int rows_total = p.group * p.q_len;
  const int row0 = rb * ROWS;
  const int rows_here = min(ROWS, rows_total - row0);
  const int tok_max = (row0 + rows_here - 1) / p.group;
  long long a0, a1, b0 = 0, b1 = 0, base, slots;
  const uint8_t *gk, *gv;
  const __half *gks, *gkz, *gvs, *gvz;
  if (is_full) {
    base = p.full_len;
    const long long nkeys = p.full_len + tok_max + 1;
    a0 = (long long)split * p.keys_per_split;
    a1 = min(nkeys, a0 + (long long)p.keys_per_split);
    if (a1 < a0) a1 = a0;
    slots = p.full_cap;
    const long long hrow = ((long long)b * p.n_full + kvh) * p.full_cap;
    gk = p.full_k + hrow * 64;
    gv = p.full_v + hrow * 64;
    gks = p.fks + hrow;
    gkz = p.fkz + hrow;
    gvs = p.fvs + hrow;
    gvz = p.fvz + hrow;
  } else {
    base = p.stage_off;
    a0 = 0;
    a1 = p.cache_scan;
    b0 = p.stage_off;
    b1 = (long long)p.stage_off + tok_max + 1;
    slots = p.ring_slots;
    const long long hrow = ((long long)b * p.n_stream + (kvh - p.n_full)) * p.ring_slots;
    gk = p.ring_k + hrow * 64;
    gv = p.ring_v + hrow * 64;
    gks = p.rks + hrow;
    gkz = p.rkz + hrow;
    gvs = p.rvs + hrow;
    gvz = p.rvz + hrow;
  }
  const int nA = (int)((a1 - a0 + I4_TILE - 1) / I4_TILE);
  const int nB = (int)((b1 - b0 + I4_TILE - 1) / I4_TILE);
  const int n_tiles = nA + nB;
  auto tile_start = [&](int i) -> long long {
    return i < nA ? a0 + (long long)i * I4_TILE : b0 + (long long)(i - nA) * I4_TILE;
  };
  auto tile_end = [&](int i) -> long long { return i < nA ? a1 : b1; };

  // ---- cooperative tile loader: 16 B cp.async, zero-fill for rows past the segment / allocation ----
  auto issue = [&](int i) {
    if (i < n_tiles) {
      const long long j0 = tile_start(i);
      const long long lim = min(tile_end(i), slots);  // rows >= lim are not read (zero-filled)
      const uint32_t sbase = smem_u32(smem + (i % I4_STAGES) * I4_STAGE_BYTES);
      {
        if (j0 + I4_TILE <= lim) {  // interior tile: one address per thread, immediate offsets, no predicates
          const int r0 = tid >> 2, c = tid & 3;
          const uint32_t doff = r0 * 64 + ((c ^ ((r0 >> 1) & 3)) << 4);
          const long long off = (j0 + r0) * 64 + c * 16;
#pragma unroll
          for (int it = 0; it < I4_TILE * 4 / I4_THREADS; ++it) {
            cp_async16(sbase + doff + it * 2048, gk + off + it * 2048, 16);
            cp_async16(sbase + I4_PACK_BYTES + doff + it * 2048, gv + off + it * 2048, 16);
          }
          if (tid < I4_TILE / 2) {
            constexpr int CPA = I4_TILE / 8;
            const int arr = tid / CPA, qd = tid % CPA;
            const __half* src = arr == 0 ? gks : arr == 1 ? gkz : arr == 2 ? gvs : gvz;
            cp_async16(sbase + 2 * I4_PACK_BYTES + arr * (I4_TILE * 2) + qd * 16, src + j0 + qd * 8, 16);
          }
          cp_async_commit();
          return;
        }
      }
#pragma unroll
      for (int it = 0; it < I4_TILE * 4 / I4_THREADS; ++it) {
        const int chunk = tid + it * I4_THREADS;  // row = chunk/4, c = chunk%4
        const int r = chunk >> 2, c = chunk & 3;
        const bool ok = (j0 + r) < lim;
        const long long srow = ok ? (j0 + r) : 0;
        const uint32_t doff = r * 64 + ((c ^ ((r >> 1) & 3)) << 4);
        cp_async16(sbase + doff, gk + srow * 64 + c * 16, ok ? 16 : 0);
        cp_async16(sbase + I4_PACK_BYTES + doff, gv + srow * 64 + c * 16, ok ? 16 : 0);
      }
      if (tid < I4_TILE / 2) {
        constexpr int CPA = I4_TILE / 8;          // 16-byte chunks per scale/zero array
        const int arr = tid / CPA, qd = tid % CPA;  // 4 arrays x CPA chunks of 8 rows
        const __half* src = arr == 0 ? gks : arr == 1 ? gkz : arr == 2 ? gvs : gvz;
        const long long r0 = j0 + qd * 8;
        long long nb = (lim - r0) * 2;
        nb = nb < 0 ? 0 : (nb > 16 ? 16 : nb);
        cp_async16(sbase + 2 * I4_PACK_BYTES + arr * (I4_TILE * 2) + qd * 16, src + (nb > 0 ? r0 : 0), (int)nb);
      }
    }
    cp_async_commit();
  };
#pragma unroll
  for (int i = 0; i < I4_STAGES - 1; ++i) issue(i);

  // ---- Q fragments in the permuted head_dim order + per-row offsets ------------------------------
  const int wrow = (KEY_WARPS == 1) ? warp * 16 : 0;
  const int wkey = (KEY_WARPS == 1) ? 0 : warp * KPW;
  uint32_t qa[8][4];
  int tok_r[2];
  float qsum[2], qoff[2];
  {
    const T* qb = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_batch_stride;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int R = row0 + wrow + g + hf * 8;
      const bool ok = R < rows_total;
      const int tok = ok ? R / p.group : 0;
      const int hq = kvh * p.group + (ok ? R % p.group : 0);
      tok_r[hf] = ok ? tok : -1;
      const T* src = qb + (long long)tok * p.q_tok_stride + (long long)hq * kHeadDim + 32 * t4;
      float s_all = 0.f, s_off = 0.f;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        __half e[8];
        if (ok) {
          if constexpr (std::is_same<T, __half>::value) {
            *reinterpret_cast<uint4*>(e) = *reinterpret_cast<const uint4*>(src + 8 * w);
          } else {
            T et[8];
            *reinterpret_cast<uint4*>(et) = *reinterpret_cast<const uint4*>(src + 8 * w);
#pragma unroll
            for (int i = 0; i < 8; ++i) e[i] = to_half(et[i]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) e[i] = __float2half(0.f);
        }
        const __half sixteenth = __float2half(0.0625f);
        // lo slots carry +1024, hi slots carry Q/16 against codes*16 (+1024)
        const __half h0 = __hmul(e[0], sixteenth), h4 = __hmul(e[4], sixteenth);
        const __half h2 = __hmul(e[2], sixteenth), h6 = __hmul(e[6], sixteenth);
        qa[2 * w][hf] = Op::pack(__half2float(e[1]), __half2float(e[5]));          // k = 2t,2t+1   <- d+1, d+5
        qa[2 * w][hf + 2] = Op::pack(__half2float(h0), __half2float(h4));           // k = 2t+8,+9   <- (d+0, d+4)/16
        qa[2 * w + 1][hf] = Op::pack(__half2float(e[3]), __half2float(e[7]));      //               <- d+3, d+7
        qa[2 * w + 1][hf + 2] = Op::pack(__half2float(h2), __half2float(h6));       //               <- (d+2, d+6)/16
#pragma unroll
        for (int i = 0; i < 8; ++i) s_all += __half2float(e[i]);
        s_off += 1024.f * (__half2float(e[1]) + __half2float(e[5]) + __half2float(e[3]) + __half2float(e[7]) +
                           __half2float(h0) + __half2float(h4) + __half2float(h2) + __half2float(h6));
      }
      s_all += __shfl_xor_sync(0xffffffffu, s_all, 1);
      s_all += __shfl_xor_sync(0xffffffffu, s_all, 2);
      s_off += __shfl_xor_sync(0xffffffffu, s_off, 1);
      s_off += __shfl_xor_sync(0xffffffffu, s_off, 2);
      qsum[hf] = s_all;
      qoff[hf] = s_off;
    }
  }

  float o[16][4];  // logical n-tile (blk, i): index blk*4+i, column n <-> head_dim 32 blk + 4 n + i
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};   // sum p
  float ps_run[2] = {0.f, 0.f};  // sum fp16(p * s_v)   (offset removal)
  float pz_run[2] = {0.f, 0.f};  // sum p * z_v
  const int lrow = lane & 7, lmat = lane >> 3;

  for (int i = 0; i < n_tiles; ++i) {
    cp_async_wait<I4_STAGES - 2>();
    __syncthreads();          // tile i landed for everyone; everyone is done with tile i-1
    issue(i + I4_STAGES - 1); // refills the stage tile i-1 used
    const uint8_t* st = smem + (i % I4_STAGES) * I4_STAGE_BYTES;
    const uint32_t sK = smem_u32(st), sV = sK + I4_PACK_BYTES;
    const __half* sKs = reinterpret_cast<const __half*>(st + 2 * I4_PACK_BYTES);
    const __half* sKz = sKs + I4_TILE;
    const __half* sVs = sKs + 2 * I4_TILE;
    const __half* sVz = sKs + 3 * I4_TILE;
    const long long j0 = tile_start(i);
    const long long jend = tile_end(i);

    // ---- S_raw = Q . codes(K) ----------------------------------------------------------------------
    float sc[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
      const int key = wkey + n * 8 + g;
      const uint32_t addr = sK + key * 64 + ((t4 ^ ((key >> 1) & 3)) << 4);
      uint32_t w0, w1, w2, w3;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "r"(addr));
      const uint32_t ww[4] = {w0, w1, w2, w3};
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const uint32_t x = ww[w], y = x >> 8;
        Op::run(sc[n], qa[2 * w], lop1_lo(x), lop1_hi(x));
        Op::run(sc[n], qa[2 * w + 1], lop1_lo(y), lop1_hi(y));
      }
    }
    // ---- logits: s_j * (S_raw - qoff) + z_j * qsum, mask (boundary tiles only), online softmax --------
    const long long kfirst = j0 + wkey;
    const int tmin = (row0 + wrow) / p.group;
    const bool need_mask = (kfirst + KPW > jend) || (kfirst + KPW - 1 > base + tmin) || (!is_full && i < nA);
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const int kc = wkey + n * 8 + 2 * t4;
      const float2 ks = __half22float2(*reinterpret_cast<const __half2*>(sKs + kc));
      const float2 kz = __half22float2(*reinterpret_cast<const __half2*>(sKz + kc));
      sc[n][0] = ks.x * (sc[n][0] - qoff[0]) + kz.x * qsum[0];
      sc[n][1] = ks.y * (sc[n][1] - qoff[0]) + kz.y * qsum[0];
      sc[n][2] = ks.x * (sc[n][2] - qoff[1]) + kz.x * qsum[1];
      sc[n][3] = ks.y * (sc[n][3] - qoff[1]) + kz.y * qsum[1];
    }
    if (need_mask) {
#pragma unroll
      for (int n = 0; n < NT; ++n) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const long long j = kfirst + n * 8 + 2 * t4 + (e & 1);
          const int tk = tok_r[e >> 1];
          bool vis = (tk >= 0) && (j < jend) && (j <= base + tk);
          if (!is_full && i < nA) vis = vis && stream_slot_valid((int)j, p.sink, p.recent, p.total, p.lo);
          if (!vis) sc[n][e] = -INFINITY;
        }
      }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      mx[0] = fmaxf(mx[0], fmaxf(sc[n][0], sc[n][1]));
      mx[1] = fmaxf(mx[1], fmaxf(sc[n][2], sc[n][3]));
    }
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 1));
      mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 2));
    }
    // the running max rarely moves after the first tiles of a long context: rescale only when it does
    const bool moved = __any_sync(0xffffffffu, (mx[0] > m_run[0]) || (mx[1] > m_run[1]));
    float msc[2];
    if (moved) {
      float alpha[2];
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const float m_new = fmaxf(m_run[hf], mx[hf]);
        const float msn = (m_new == -INFINITY) ? 0.f : m_new * p.scale_log2;
        alpha[hf] = (m_run[hf] == -INFINITY) ? 0.f : fast_exp2(m_run[hf] * p.scale_log2 - msn);
        m_run[hf] = m_new;
        l_run[hf] *= alpha[hf];
        ps_run[hf] *= alpha[hf];
        pz_run[hf] *= alpha[hf];
      }
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        o[d][0] *= alpha[0];
        o[d][1] *= alpha[0];
        o[d][2] *= alpha[1];
        o[d][3] *= alpha[1];
      }
    }
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) msc[hf] = (m_run[hf] == -INFINITY) ? 0.f : m_run[hf] * p.scale_log2;
    float rs[2] = {0.f, 0.f}, rps[2] = {0.f, 0.f}, rpz[2] = {0.f, 0.f};
    uint32_t pa[NT / 2][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const int kc = wkey + n * 8 + 2 * t4;
      const float2 vs = __half22float2(*reinterpret_cast<const __half2*>(sVs + kc));
      const float2 vz = __half22float2(*reinterpret_cast<const __half2*>(sVz + kc));
      const float p0 = fast_exp2(sc[n][0] * p.scale_log2 - msc[0]);
      const float p1 = fast_exp2(sc[n][1] * p.scale_log2 - msc[0]);
      const float p2 = fast_exp2(sc[n][2] * p.scale_log2 - msc[1]);
      const float p3 = fast_exp2(sc[n][3] * p.scale_log2 - msc[1]);
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      rpz[0] += p0 * vz.x + p1 * vz.y;
      rpz[1] += p2 * vz.x + p3 * vz.y;
      const __half2 a = __floats2half2_rn(p0 * vs.x, p1 * vs.y);  // p' = p * s_v, rounded to fp16 like P
      const __half2 c = __floats2half2_rn(p2 * vs.x, p3 * vs.y);
      rps[0] += __low2float(a) + __high2float(a);
      rps[1] += __low2float(c) + __high2float(c);
      pa[n >> 1][(n & 1) * 2 + 0] = *reinterpret_cast<const uint32_t*>(&a);
      pa[n >> 1][(n & 1) * 2 + 1] = *reinterpret_cast<const uint32_t*>(&c);
    }
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      l_run[hf] += rs[hf];
      ps_run[hf] += rps[hf];
      pz_run[hf] += rpz[hf];
    }
    // ---- O_raw += P' . codes(V): ldmatrix.trans on 16-bit units (4 codes of one key) ---------------
#pragma unroll
    for (int k2 = 0; k2 < NT / 2; ++k2) {
#pragma unroll
      for (int call = 0; call < 2; ++call) {
        const int key = wkey + k2 * 16 + (lmat & 1) * 8 + lrow;
        const int blk = 2 * call + (lmat >> 1);
        const uint32_t addr = sV + key * 64 + ((blk ^ ((key >> 1) & 3)) << 4);
        uint32_t r0, r1, r2, r3;  // (keys 0-7, blk) (keys 8-15, blk) (keys 0-7, blk+1) (keys 8-15, blk+1)
        ldsm_x4_trans(r0, r1, r2, r3, addr);
        const int nb = (2 * call) * 4;
        Op::run(o[nb + 1], pa[k2], lop1_lo(r0), lop1_lo(r1));            // i = 1
        Op::run(o[nb + 0], pa[k2], lop1_hi(r0), lop1_hi(r1));            // i = 0 (x16)
        Op::run(o[nb + 3], pa[k2], lop1_lo(r0 >> 8), lop1_lo(r1 >> 8));  // i = 3
        Op::run(o[nb + 2], pa[k2], lop1_hi(r0 >> 8), lop1_hi(r1 >> 8));  // i = 2 (x16)
        Op::run(o[nb + 5], pa[k2], lop1_lo(r2), lop1_lo(r3));
        Op::run(o[nb + 4], pa[k2], lop1_hi(r2), lop1_hi(r3));
        Op::run(o[nb + 7], pa[k2], lop1_lo(r2 >> 8), lop1_lo(r3 >> 8));
        Op::run(o[nb + 6], pa[k2], lop1_hi(r2 >> 8), lop1_hi(r3 >> 8));
      }
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 1);
    l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 2);
    ps_run[hf] += __shfl_xor_sync(0xffffffffu, ps_run[hf], 1);
    ps_run[hf] += __shfl_xor_sync(0xffffffffu, ps_run[hf], 2);
    pz_run[hf] += __shfl_xor_sync(0xffffffffu, pz_run[hf], 1);
    pz_run[hf] += __shfl_xor_sync(0xffffffffu, pz_run[hf], 2);
  }

  // ---- true (un-normalised) O of this warp -> shared memory, in natural head_dim order -------------
  __syncthreads();
  float* sm_o = reinterpret_cast<float*>(smem);               // [ROWS][128] merged
  float* sm_ml = reinterpret_cast<float*>(smem + 64 * 1024);  // [ROWS][2]
  float* w_o = (KEY_WARPS == 4) ? reinterpret_cast<float*>(smem) + 16 * 128 : sm_o;  // [4][16][128] | [ROWS][128]
  float* w_ml = (KEY_WARPS == 4) ? sm_ml + 64 : sm_ml;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int r = (KEY_WARPS == 4) ? (warp * 16 + g + hf * 8) : (wrow + g + hf * 8);
    if (t4 == 0) {
      w_ml[r * 2 + 0] = (m_run[hf] == -INFINITY) ? -INFINITY : m_run[hf] * p.scale_log2;
      w_ml[r * 2 + 1] = l_run[hf];
    }
    const float off = 1024.f * ps_run[hf];
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
      const int blk = nt >> 2, ii = nt & 3;
      const float mul = (ii & 1) ? 1.f : 0.0625f;  // hi-nibble columns carry codes * 16
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int d = 32 * blk + 4 * (2 * t4 + e) + ii;
        w_o[r * 128 + d] = (o[nt][hf * 2 + e] - off) * mul + pz_run[hf];
      }
    }
  }
  __syncthreads();
  if constexpr (KEY_WARPS == 4) {
    for (int idx = tid; idx < 16 * 128; idx += I4_THREADS) {
      const int r = idx >> 7, d = idx & 127;
      float mm = -INFINITY;
#pragma unroll
      for (int w = 0; w < 4; ++w) mm = fmaxf(mm, w_ml[(w * 16 + r) * 2]);
      float acc = 0.f, ll = 0.f;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const float mw = w_ml[(w * 16 + r) * 2];
        const float f = (mw == -INFINITY) ? 0.f : fast_exp2(mw - mm);
        acc += f * w_o[(w * 16 + r) * 128 + d];
        ll += f * w_ml[(w * 16 + r) * 2 + 1];
      }
      sm_o[r * 128 + d] = acc;
      if (d == 0) {
        sm_ml[r * 2] = mm;
        sm_ml[r * 2 + 1] = ll;
      }
    }
    __syncthreads();
  }

  T* outb = reinterpret_cast<T*>(p.out) + (long long)b * p.out_batch_stride;
  auto store_row_elem = [&](int r, int d, float v0, float v1) {
    const int R = row0 + r;
    const int tok = R / p.group;
    const int hq = kvh * p.group + R % p.group;
    T* dst = outb + ((long long)tok * p.n_q_heads + hq) * kHeadDim + d;
    *reinterpret_cast<uint32_t*>(dst) = MmaOp<T>::pack(v0, v1);
  };
  const int nsplit = is_full ? p.splits_full : 1;
  if (nsplit == 1) {
    for (int idx = tid; idx < rows_here * 64; idx += I4_THREADS) {
      const int r = idx >> 6, d = (idx & 63) * 2;
      const float l = sm_ml[r * 2 + 1];
      const float inv = l > 0.f ? 1.f / l : 0.f;
      store_row_elem(r, d, sm_o[r * 128 + d] * inv, sm_o[r * 128 + d + 1] * inv);
    }
    return;
  }
  // ---- split-KV publish + hierarchical merge (protocol of attn_mma.cu: split_kv_finish) ---------------------------
  const long long item = ((long long)b * p.n_full + kvh) * p.n_rb + rb;
  float* wo = p.ws.ws_o + (item * p.splits_full + split) * (long long)(ROWS * 128);
  float* wml = p.ws.ws_ml + (item * p.splits_full + split) * (long long)(ROWS * 2);
  for (int idx = tid; idx < rows_here * 32; idx += I4_THREADS) {
    const int r = idx >> 5, d4 = (idx & 31) * 4;
    *reinterpret_cast<float4*>(&wo[r * 128 + d4]) = *reinterpret_cast<const float4*>(&sm_o[r * 128 + d4]);
  }
  if (tid < rows_here * 2) wml[tid] = sm_ml[tid];
  split_kv_finish<ROWS>(p.ws, item, split, p.splits_full, rows_here, reinterpret_cast<float*>(smem),
                        reinterpret_cast<float*>(smem + 80 * 1024), &s_is_last,
                        [&](int r, int d, float v0, float v1, float, float) { store_row_elem(r, d, v0, v1); });
}

// =============================================================================================
// Decode variant with the operand roles swapped ("keys are M"): S^T = codes(K) . Q^T and O^T = codes(V)^T . P'^T.
//
// With group * q_len <= 8 query rows, the row-major formulation above pads them to the 16-row M dimension of
// m16n8k16 (4 useful rows of 16 for a GQA-4 decode step).  Here the 16 KEYS of an m-tile are M and the query rows
// are the 8-wide N dimension, which halves the HMMA count (34 instead of 64 per warp per 32 keys), the logits /
// exponentials per thread (8 instead of 16) and the accumulator registers (32 instead of 64), so four CTAs fit on
// an SM instead of two.  The nibble -> fp16 conversion is unchanged (the same LOP3 results now fill A fragments:
// the A row-major and B col-major fragments of m16n8k16 map threads identically).  S^T leaves the QK^T product
// in (key g | rows 2t,2t+1) order; P'^T must enter the PV product as (keys 2t,2t+1 | row g): one
// movmatrix.trans per 8 keys.  sum_j fp16(p'_j) (the +1024 offset removal) is one extra HMMA against a
// constant-one A fragment per 16 keys instead of unpack+add on the ALU pipe, and the running-max reduction
// across lanes is only executed on tiles where some lane saw a logit above the running max.
//
// The fragment algebra is also checked lane-by-lane on the CPU
// (tests/test_int4_swapab_layout.py).
// =============================================================================================
// Debug build only (`make trace`, -DDUO_TRACE): per-CTA %globaltimer stamps (start, main loop done, partial published,
// exit) into a caller-provided buffer, from which a launch timeline can be drawn.
#ifdef DUO_TRACE
__device__ unsigned long long* g_duo_trace = nullptr;
__device__ __forceinline__ void trace_stamp(int slot) {
  if (threadIdx.x == 0 && g_duo_trace) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_duo_trace[((long long)blockIdx.y * gridDim.x + blockIdx.x) * 4 + slot] = t;
  }
}
#define DUO_TRACE_STAMP(slot) trace_stamp(slot)
#else
#define DUO_TRACE_STAMP(slot)
#endif

constexpr int D8_TILE = 128;
constexpr int D8_STAGES = 3;
constexpr int D8_PACK = D8_TILE * 64;
constexpr int D8_STAGE_BYTES = 2 * D8_PACK + 4 * D8_TILE * 2;
constexpr int D8_ROWS = 8;
constexpr int D8_SMEM_BYTES = D8_STAGES * D8_STAGE_BYTES + 128;
static_assert(D8_STAGES * D8_STAGE_BYTES >= (4 * D8_ROWS * 128 + D8_ROWS * 128 + 5 * D8_ROWS * 2) * 4, "merge smem");

__device__ __forceinline__ float lds_half(uint32_t addr) {
  unsigned short h;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(addr));
  return __half2float(__ushort_as_half(h));
}
__device__ __forceinline__ uint32_t movm_trans(uint32_t a) {
  uint32_t d;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(d) : "r"(a));
  return d;
}

// RAGGED (FUSED only): one launch decodes a batch whose rows have different lengths.  The grid is n_full * rg_slots
// retrieval slots (kv-head major), then batch * n_stream streaming CTAs; every retrieval CTA derives the batch's key
// partition from row_state (dec8 policy: 128-key tiles, >= 1024 keys per split, nkeys = full_len + q_len per row) and
// finds its row and split.  Idle slots exit before any load.
// SEQ: the retrieval cache is this rank's slice of a sequence-sharded cache (see I4Params).  The key range of a
// retrieval head is its local rows of positions < full_len + q_len (dec8 split policy on those); token t sees the local
// rows of positions <= full_len + t, and a slice is in position order, so no other mask applies.  FUSED (one token):
// only the owner of position full_len quantises the new K / V, into its next local row.
template <bool FUSED, typename T, bool RAGGED = false, bool POOLED = false, bool SEQ = false>
__global__ void __launch_bounds__(I4_THREADS, 4) duo_attn_int4_dec8_kernel(const I4Params pin) {
  static_assert(!RAGGED || FUSED, "the ragged variant is the fused decode kernel");
  static_assert(!POOLED || RAGGED, "the pooled layout is a ragged decode layout");
  static_assert(!SEQ || !RAGGED, "sequence sharding is not combined with the ragged layouts");
  DUO_TRACE_STAMP(0);
  I4Params p = pin;
  if (!RAGGED && pin.dstate) {
    p.full_len = pin.dstate[0];
    p.total = pin.dstate[1];
    p.lo = pin.dstate[2];
    const long long nk = p.full_len + p.q_len;
    p.keys_per_split = (int)split_keys(SEQ ? seq_local_len(nk, p.seq_rank, p.seq_world, p.seq_block) : nk,
                                       p.splits_full, D8_TILE);
    p.cache_scan = (int)(p.total < p.W ? p.total : p.W);
  }
  constexpr int KPW = 32;  // keys per warp per tile
  using Op = MmaOp<__half>;

  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  __shared__ int s_is_last;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  int b = blockIdx.y;

  const int n_full_items = p.n_full * p.splits_full;
  int kvh, split;
  bool is_full;
  if constexpr (RAGGED) {
    const long long* rs = pin.dstate;
    split = 0;
    const int x = blockIdx.x, n_fslots = p.n_full * p.rg_slots;
    is_full = x < n_fslots;
    if (is_full) {
      // the new tokens are rows full_len + t of the cache: row b's key range is full_len + q_len keys
      const long long kps = ragged_batch_kps(rs, p.batch, p.q_len, p.rg_want, D8_TILE, 8 * D8_TILE);
      kvh = x / p.rg_slots;
      const RaggedSlot s = ragged_slot(rs, p.batch, p.q_len, kps, x % p.rg_slots);
      b = s.b;
      if (b == p.batch) return;  // idle slot
      split = s.split;
      p.keys_per_split = (int)kps;
      p.splits_full = s.splits;
      ragged_ws_slice<D8_ROWS>(p.ws, b, kvh, p.n_full, p.rg_slots, s);
    } else {
      const int y = x - n_fslots;
      b = y / p.n_stream;
      kvh = p.n_full + y % p.n_stream;
    }
    p.full_len = rs[4 * b];
    p.total = rs[4 * b + 1];
    p.lo = rs[4 * b + 2];
    p.cache_scan = (int)(p.total < p.W ? p.total : p.W);
    // per-row RoPE tables [batch][q_len][128]
    const long long tab = (long long)b * p.q_len * kHeadDim * (p.rope_mode == DUO_ROPE_HF ? (long long)sizeof(T) : 4);
    p.cos = reinterpret_cast<const uint8_t*>(p.cos) + tab;
    p.sin = reinterpret_cast<const uint8_t*>(p.sin) + tab;
  } else if ((int)blockIdx.x < n_full_items) {
    is_full = true;
    split = blockIdx.x % p.splits_full;
    kvh = blockIdx.x / p.splits_full;
  } else {
    is_full = false;
    kvh = p.n_full + (blockIdx.x - n_full_items);
    split = 0;
  }
  const int rows_total = p.group * p.q_len;  // <= 8
  const int tok_max = (rows_total - 1) / p.group;
  long long a0, a1, b0 = 0, b1 = 0, base, slots;
  const uint8_t *gk, *gv;
  const __half *gks, *gkz, *gvs, *gvz;
  // SEQ, FUSED: this rank's local rows of positions < full_len, and whether it owns position full_len (the new token,
  // which then goes to local row seq_loc)
  long long seq_loc = 0;
  bool seq_own = false;
  if constexpr (SEQ && FUSED) {
    seq_loc = seq_local_len(p.full_len, p.seq_rank, p.seq_world, p.seq_block);
    seq_own = (int)((p.full_len / p.seq_block) % p.seq_world) == p.seq_rank;
  }
  if (is_full) {
    // SEQ: key j is visible to token t iff j < seq_local_len(full_len + t + 1); `base` (the last key token 0 sees) only
    // decides which tiles take the mask
    base = !SEQ ? p.full_len
           : FUSED ? seq_loc + seq_own - 1
                   : seq_local_len(p.full_len + 1, p.seq_rank, p.seq_world, p.seq_block) - 1;
    const long long nkeys = !SEQ  ? p.full_len + tok_max + 1
                            : FUSED ? seq_loc + seq_own
                                    : seq_local_len(p.full_len + tok_max + 1, p.seq_rank, p.seq_world, p.seq_block);
    a0 = (long long)split * p.keys_per_split;
    a1 = min(nkeys, a0 + (long long)p.keys_per_split);
    if (a1 < a0) a1 = a0;
    long long hrow;
    if constexpr (POOLED) {  // row b's region: pool rows first_b * n_full + kvh * cap_b + j
      slots = pin.row_geom[2 * b + 1];
      hrow = pin.row_geom[2 * b] * p.n_full + kvh * slots;
    } else {
      slots = p.full_cap;
      hrow = ((long long)b * p.n_full + kvh) * p.full_cap;
    }
    gk = p.full_k + hrow * 64;
    gv = p.full_v + hrow * 64;
    gks = p.fks + hrow;
    gkz = p.fkz + hrow;
    gvs = p.fvs + hrow;
    gvz = p.fvz + hrow;
  } else {
    base = p.stage_off;
    a0 = 0;
    a1 = p.cache_scan;
    b0 = p.stage_off;
    b1 = (long long)p.stage_off + tok_max + 1;
    slots = p.ring_slots;
    const long long hrow = ((long long)b * p.n_stream + (kvh - p.n_full)) * p.ring_slots;
    gk = p.ring_k + hrow * 64;
    gv = p.ring_v + hrow * 64;
    gks = p.rks + hrow;
    gkz = p.rkz + hrow;
    gvs = p.rvs + hrow;
    gvz = p.rvz + hrow;
  }
  const int nA = (int)((a1 - a0 + D8_TILE - 1) / D8_TILE);
  const int nB = (int)((b1 - b0 + D8_TILE - 1) / D8_TILE);
  const int n_tiles = nA + nB;
  auto tile_start = [&](int i) -> long long {
    return i < nA ? a0 + (long long)i * D8_TILE : b0 + (long long)(i - nA) * D8_TILE;
  };
  auto tile_end = [&](int i) -> long long { return i < nA ? a1 : b1; };

  // loader: same tile image as duo_attn_int4_kernel<4>.  Interior tiles (every row valid) take a path with one
  // address per thread and immediate offsets; boundary tiles predicate and zero-fill per row.
  const int ld_r0 = tid >> 2, ld_c = tid & 3;
  const uint32_t ld_doff = ld_r0 * 64 + ((ld_c ^ ((ld_r0 >> 1) & 3)) << 4);
  const int ld_arr = (tid & 63) >> 4, ld_qd = tid & 15;  // scale/zero arrays: 4 arrays x 16 chunks of 8 rows
  const __half* ld_src = ld_arr == 0 ? gks : ld_arr == 1 ? gkz : ld_arr == 2 ? gvs : gvz;
  const uint32_t ld_soff = 2 * D8_PACK + ld_arr * (D8_TILE * 2) + ld_qd * 16;
  auto issue = [&](int i) {
    if (i < n_tiles) {
      const long long j0 = tile_start(i);
      const long long lim = min(tile_end(i), slots);  // rows >= lim are not read (zero-filled)
      const uint32_t sbase = smem_u32(smem + (i % D8_STAGES) * D8_STAGE_BYTES);
      if (j0 + D8_TILE <= lim) {
        const long long off = (j0 + ld_r0) * 64 + ld_c * 16;
        const uint8_t* kp = gk + off;
        const uint8_t* vp = gv + off;
#pragma unroll
        for (int it = 0; it < D8_TILE * 4 / I4_THREADS; ++it) {
          cp_async16(sbase + ld_doff + it * 2048, kp + it * 2048, 16);
          cp_async16(sbase + D8_PACK + ld_doff + it * 2048, vp + it * 2048, 16);
        }
        if (tid < D8_TILE / 2) cp_async16(sbase + ld_soff, ld_src + j0 + ld_qd * 8, 16);
      } else {
#pragma unroll
        for (int it = 0; it < D8_TILE * 4 / I4_THREADS; ++it) {
          const int r = ld_r0 + it * 32;
          const bool ok = (j0 + r) < lim;
          const long long srow = ok ? (j0 + r) : 0;
          cp_async16(sbase + ld_doff + it * 2048, gk + srow * 64 + ld_c * 16, ok ? 16 : 0);
          cp_async16(sbase + D8_PACK + ld_doff + it * 2048, gv + srow * 64 + ld_c * 16, ok ? 16 : 0);
        }
        if (tid < D8_TILE / 2) {
          const long long r0 = j0 + ld_qd * 8;
          long long nb = (lim - r0) * 2;
          nb = nb < 0 ? 0 : (nb > 16 ? 16 : nb);
          cp_async16(sbase + ld_soff, ld_src + (nb > 0 ? r0 : 0), (int)nb);
        }
      }
    }
    cp_async_commit();
  };
  // FUSED: the new tokens — RoPE(K) and K1 quantisation of K and V into the rows this CTA is about to read (retrieval
  // heads: cache rows full_len + t, written by the split whose key range holds them; streaming heads: the staging rows).
  // SEQ (one token): only the owner of position full_len writes, into local row seq_local_len(full_len)
  // = (full_len / (block * world)) * block + full_len % block; the other ranks' retrieval caches are not touched.
  auto append_new = [&]() {
    // one warp per (token, K|V) row, arithmetic of rope_append_kernel (kv_ops.cu) => the same bits as the unfused path
    const T* rows = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_batch_stride;
    for (int w = warp; w < 2 * p.q_len; w += I4_THREADS / 32) {
      const int t = w >> 1;
      const bool is_k = (w & 1) == 0;
      long long dr;  // destination row inside this head's cache
      if (is_full) {
        dr = p.full_len + t;
        if constexpr (SEQ) {
          if (!seq_own) continue;
          dr = seq_loc + t;
        }
        if (dr < a0 || dr >= a1) continue;  // another split owns (and reads) this row
      } else {
        dr = (long long)p.stage_off + t;
      }
      const T* src = rows + (long long)t * p.q_tok_stride + (is_k ? p.k_off : p.v_off) + (long long)kvh * kHeadDim;
      Vec4<T> xv = *reinterpret_cast<const Vec4<T>*>(src + lane * 4);
      if (is_k && p.rope_mode != DUO_ROPE_NONE) rope_row4<T>(xv, lane, t, p.cos, p.sin, p.rope_mode);
      float xo[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) xo[i] = RopeCvt<T>::to_f(xv.v[i]);
      quant_row_int4(xo, lane, const_cast<uint8_t*>(is_k ? gk : gv) + dr * 64,
                     const_cast<__half*>(is_k ? gks : gvs) + dr, const_cast<__half*>(is_k ? gkz : gvz) + dr);
    }
    __threadfence();
    __syncthreads();  // the rows are in memory before any cp.async of this CTA may fetch them
  };
  // The first STAGES - 1 tiles are fetched before the new rows are produced (their loads fly meanwhile) unless one of
  // them already holds a new row (short key ranges).
  bool append_first = false;
  if constexpr (FUSED)
    append_first = is_full ? (a0 + (long long)(D8_STAGES - 1) * D8_TILE > p.full_len) : (nA < D8_STAGES - 1);
  if constexpr (FUSED && SEQ) {  // the new row is local row seq_loc
    if (is_full) append_first = a0 + (long long)(D8_STAGES - 1) * D8_TILE > seq_loc;
  }
  if constexpr (FUSED) {
    if (append_first) append_new();
  }
#pragma unroll
  for (int i = 0; i < D8_STAGES - 1; ++i) issue(i);
  if constexpr (FUSED) {
    if (!append_first) append_new();
  }

  // ---- Q^T as B fragments: lane (g, t4) holds query row g, head_dim chunk 32 t4 .. 32 t4 + 31 ------------
  const int wkey = warp * KPW;
  uint32_t qb[8][2];
  float qsum[2], qoff[2];
  int tok_r[2];
  long long vis_r[2];  // SEQ, several tokens: keys of the slice visible to the query rows of this lane
  {
    const T* qbase = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_batch_stride;
    const bool ok = g < rows_total;
    const int tok = ok ? g / p.group : 0;
    const int hq = kvh * p.group + (ok ? g % p.group : 0);
    const T* src = qbase + (long long)tok * p.q_tok_stride + (long long)hq * kHeadDim + 32 * t4;
    float s_all = 0.f, s_off = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      __half e[8];
      if (ok) {
        // RoPE in the activation type T, then (bf16) round to the fp16 of the fragments
        T* et = reinterpret_cast<T*>(e);
        T eb[std::is_same<T, __half>::value ? 1 : 8];
        if constexpr (!std::is_same<T, __half>::value) et = eb;
        *reinterpret_cast<uint4*>(et) = *reinterpret_cast<const uint4*>(src + 8 * w);
        if constexpr (FUSED) {
          if (p.rope_mode != DUO_ROPE_NONE) {  // partner of head_dim d is d +- 64: the chunk of lane t4 ^ 2
            uint4 mine = *reinterpret_cast<const uint4*>(et);
            uint4 other = *reinterpret_cast<const uint4*>(src + 8 * w + (t4 < 2 ? 64 : -64));
            if (t4 < 2) {
              rope8<T>(mine, other, p.cos, p.sin, p.rope_mode, tok, 32 * t4 + 8 * w);
            } else {
              rope8<T>(other, mine, p.cos, p.sin, p.rope_mode, tok, 32 * (t4 - 2) + 8 * w);
            }
            *reinterpret_cast<uint4*>(et) = mine;
          }
        }
        if constexpr (!std::is_same<T, __half>::value) {
#pragma unroll
          for (int i = 0; i < 8; ++i) e[i] = to_half(eb[i]);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) e[i] = __float2half(0.f);
      }
      const __half sixteenth = __float2half(0.0625f);
      const __half h0 = __hmul(e[0], sixteenth), h4 = __hmul(e[4], sixteenth);
      const __half h2 = __hmul(e[2], sixteenth), h6 = __hmul(e[6], sixteenth);
      qb[2 * w][0] = Op::pack(__half2float(e[1]), __half2float(e[5]));      // k = 2t,2t+1   <- d+1, d+5
      qb[2 * w][1] = Op::pack(__half2float(h0), __half2float(h4));          // k = 2t+8,+9   <- (d+0, d+4)/16
      qb[2 * w + 1][0] = Op::pack(__half2float(e[3]), __half2float(e[7]));  //               <- d+3, d+7
      qb[2 * w + 1][1] = Op::pack(__half2float(h2), __half2float(h6));      //               <- (d+2, d+6)/16
#pragma unroll
      for (int i = 0; i < 8; ++i) s_all += __half2float(e[i]);
      s_off += 1024.f * (__half2float(e[1]) + __half2float(e[5]) + __half2float(e[3]) + __half2float(e[7]) +
                         __half2float(h0) + __half2float(h4) + __half2float(h2) + __half2float(h6));
    }
    s_all += __shfl_xor_sync(0xffffffffu, s_all, 1);
    s_all += __shfl_xor_sync(0xffffffffu, s_all, 2);
    s_off += __shfl_xor_sync(0xffffffffu, s_off, 1);
    s_off += __shfl_xor_sync(0xffffffffu, s_off, 2);
#pragma unroll
    for (int e = 0; e < 2; ++e) {  // accumulator columns of this lane are query rows 2 t4, 2 t4 + 1
      const int r = 2 * t4 + e;
      qsum[e] = __shfl_sync(0xffffffffu, s_all, r * 4);
      qoff[e] = __shfl_sync(0xffffffffu, s_off, r * 4);
      tok_r[e] = r < rows_total ? r / p.group : -1;
      if constexpr (SEQ && !FUSED)
        vis_r[e] = r < rows_total ? seq_local_len(p.full_len + r / p.group + 1, p.seq_rank, p.seq_world, p.seq_block) : 0;
    }
  }

  float oT[8][4];  // tile call*4 + i: rows of the tile are head_dim 32 (2 call) + 4 g + i  and  32 (2 call + 1) + 4 g + i
#pragma unroll
  for (int i = 0; i < 8; ++i) oT[i][0] = oT[i][1] = oT[i][2] = oT[i][3] = 0.f;
  float psT[4] = {0.f, 0.f, 0.f, 0.f};  // sum_j fp16(p'_j) per query row, from the constant-one HMMA
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};   // per-lane partial of sum p      (keys = g mod 8)
  float pz_run[2] = {0.f, 0.f};  // per-lane partial of sum p z_v
  const uint32_t ones[4] = {0x3C003C00u, 0x3C003C00u, 0x3C003C00u, 0x3C003C00u};
  const int lrow = lane & 7, lmat = lane >> 3;

  for (int i = 0; i < n_tiles; ++i) {
    cp_async_wait<D8_STAGES - 2>();
    __syncthreads();
    issue(i + D8_STAGES - 1);
    const uint8_t* st = smem + (i % D8_STAGES) * D8_STAGE_BYTES;
    const uint32_t sK = smem_u32(st), sV = sK + D8_PACK;
    const uint32_t sKs = sK + 2 * D8_PACK, sKz = sKs + 2 * D8_TILE, sVs = sKs + 4 * D8_TILE, sVz = sKs + 6 * D8_TILE;
    const long long j0 = tile_start(i);
    const long long jend = tile_end(i);

    // ---- S^T_raw = codes(K) . Q^T : 2 m-tiles of 16 keys ----------------------------------------------------
    float sc[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      sc[mt][0] = sc[mt][1] = sc[mt][2] = sc[mt][3] = 0.f;
      const int key0 = wkey + mt * 16 + g, key1 = key0 + 8;
      const uint32_t addr0 = sK + key0 * 64 + ((t4 ^ ((key0 >> 1) & 3)) << 4);
      const uint32_t addr1 = sK + key1 * 64 + ((t4 ^ ((key1 >> 1) & 3)) << 4);
      uint32_t x[4], y[4];
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x[0]), "=r"(x[1]), "=r"(x[2]), "=r"(x[3]) : "r"(addr0));
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(y[0]), "=r"(y[1]), "=r"(y[2]), "=r"(y[3]) : "r"(addr1));
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const uint32_t xl = x[w], yl = y[w], xh = xl >> 8, yh = yl >> 8;
        const uint32_t fa[4] = {lop1_lo(xl), lop1_lo(yl), lop1_hi(xl), lop1_hi(yl)};
        Op::run(sc[mt], fa, qb[2 * w][0], qb[2 * w][1]);
        const uint32_t fb[4] = {lop1_lo(xh), lop1_lo(yh), lop1_hi(xh), lop1_hi(yh)};
        Op::run(sc[mt], fb, qb[2 * w + 1][0], qb[2 * w + 1][1]);
      }
    }
    // ---- logits s_j (S_raw - qoff) + z_j qsum; mask on boundary tiles -----------------------------------------
    const long long kfirst = j0 + wkey;
    const bool need_mask = (kfirst + KPW > jend) || (kfirst + KPW - 1 > base) || (!is_full && i < nA);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
      for (int hk = 0; hk < 2; ++hk) {
        const int key = wkey + mt * 16 + hk * 8 + g;
        const float ks = lds_half(sKs + 2 * key), kz = lds_half(sKz + 2 * key);
        // the two query rows of this lane as one packed pair: ks * (S_raw - qoff) + kz * qsum
        float d0, d1, z0, z1;
        add2(d0, d1, sc[mt][hk * 2], sc[mt][hk * 2 + 1], -qoff[0], -qoff[1]);
        mul2(z0, z1, qsum[0], qsum[1], kz, kz);
        fma2(sc[mt][hk * 2], sc[mt][hk * 2 + 1], d0, d1, ks, ks, z0, z1);
      }
    }
    if (need_mask) {
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
        for (int hk = 0; hk < 2; ++hk) {
          const long long j = kfirst + mt * 16 + hk * 8 + g;
          bool kvis = j < jend;
          if (!is_full && i < nA) kvis = kvis && stream_slot_valid((int)j, p.sink, p.recent, p.total, p.lo);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int tk = tok_r[e];
            if (!(kvis && tk >= 0 && j <= base + tk)) sc[mt][hk * 2 + e] = -INFINITY;
            // SEQ: base + tk >= the last key token tk sees, so the test above keeps a superset; it is exact for one
            // token (FUSED)
            if constexpr (SEQ && !FUSED) {
              if (is_full && j >= vis_r[e]) sc[mt][hk * 2 + e] = -INFINITY;
            }
          }
        }
      }
    }
    // ---- running max: cross-lane reduction only when some lane saw a logit above it ----------------------------
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      mx[0] = fmaxf(mx[0], fmaxf(sc[mt][0], sc[mt][2]));
      mx[1] = fmaxf(mx[1], fmaxf(sc[mt][1], sc[mt][3]));
    }
    const bool moved = __any_sync(0xffffffffu, (mx[0] > m_run[0]) || (mx[1] > m_run[1]));
    if (moved) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 4));
        mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 8));
        mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 16));
      }
      float alpha[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float m_new = fmaxf(m_run[e], mx[e]);
        const float msn = (m_new == -INFINITY) ? 0.f : m_new * p.scale_log2;
        alpha[e] = (m_run[e] == -INFINITY) ? 0.f : fast_exp2(m_run[e] * p.scale_log2 - msn);
        m_run[e] = m_new;
        l_run[e] *= alpha[e];
        pz_run[e] *= alpha[e];
        psT[e] *= alpha[e];
        psT[e + 2] *= alpha[e];
      }
#pragma unroll
      for (int d = 0; d < 8; ++d) {
        oT[d][0] *= alpha[0];
        oT[d][1] *= alpha[1];
        oT[d][2] *= alpha[0];
        oT[d][3] *= alpha[1];
      }
    }
    float msc[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) msc[e] = (m_run[e] == -INFINITY) ? 0.f : m_run[e] * p.scale_log2;
    // ---- p = 2^(s - m), p' = fp16(p s_v); transpose to the B-fragment order --------------------------------------
    uint32_t pb[2][2];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
      for (int hk = 0; hk < 2; ++hk) {
        const int key = wkey + mt * 16 + hk * 8 + g;
        const float vs = lds_half(sVs + 2 * key), vz = lds_half(sVz + 2 * key);
        float x0, x1, a0, a1;
        fma2(x0, x1, sc[mt][hk * 2 + 0], sc[mt][hk * 2 + 1], p.scale_log2, p.scale_log2, -msc[0], -msc[1]);
        const float p0 = fast_exp2(x0);
        const float p1 = fast_exp2(x1);
        add2(l_run[0], l_run[1], l_run[0], l_run[1], p0, p1);
        fma2(pz_run[0], pz_run[1], p0, p1, vz, vz, pz_run[0], pz_run[1]);
        mul2(a0, a1, p0, p1, vs, vs);
        const __half2 a = __floats2half2_rn(a0, a1);  // (key | rows 2t, 2t+1)
        pb[mt][hk] = movm_trans(*reinterpret_cast<const uint32_t*>(&a));  // -> (keys 2t, 2t+1 | row g)
      }
    }
    // ---- O^T_raw += codes(V)^T . P'^T ------------------------------------------------------------------------------
#pragma unroll
    for (int k2 = 0; k2 < 2; ++k2) {
      Op::run(psT, ones, pb[k2][0], pb[k2][1]);
#pragma unroll
      for (int call = 0; call < 2; ++call) {
        const int key = wkey + k2 * 16 + (lmat & 1) * 8 + lrow;
        const int blk = 2 * call + (lmat >> 1);
        const uint32_t addr = sV + key * 64 + ((blk ^ ((key >> 1) & 3)) << 4);
        uint32_t r0, r1, r2, r3;  // (keys 0-7, blk 2c) (keys 8-15, blk 2c) (keys 0-7, blk 2c+1) (keys 8-15, blk 2c+1)
        ldsm_x4_trans(r0, r1, r2, r3, addr);
        const uint32_t h0 = r0 >> 8, h1 = r1 >> 8, h2 = r2 >> 8, h3 = r3 >> 8;
        const uint32_t f1[4] = {lop1_lo(r0), lop1_lo(r2), lop1_lo(r1), lop1_lo(r3)};
        Op::run(oT[call * 4 + 1], f1, pb[k2][0], pb[k2][1]);  // i = 1
        const uint32_t f0[4] = {lop1_hi(r0), lop1_hi(r2), lop1_hi(r1), lop1_hi(r3)};
        Op::run(oT[call * 4 + 0], f0, pb[k2][0], pb[k2][1]);  // i = 0 (x16)
        const uint32_t f3[4] = {lop1_lo(h0), lop1_lo(h2), lop1_lo(h1), lop1_lo(h3)};
        Op::run(oT[call * 4 + 3], f3, pb[k2][0], pb[k2][1]);  // i = 3
        const uint32_t f2[4] = {lop1_hi(h0), lop1_hi(h2), lop1_hi(h1), lop1_hi(h3)};
        Op::run(oT[call * 4 + 2], f2, pb[k2][0], pb[k2][1]);  // i = 2 (x16)
      }
    }
  }
  cp_async_wait<0>();
  DUO_TRACE_STAMP(1);

#pragma unroll
  for (int e = 0; e < 2; ++e) {
#pragma unroll
    for (int sh = 4; sh <= 16; sh <<= 1) {
      l_run[e] += __shfl_xor_sync(0xffffffffu, l_run[e], sh);
      pz_run[e] += __shfl_xor_sync(0xffffffffu, pz_run[e], sh);
    }
  }

  // ---- true (un-normalised) O of this warp -> shared memory in natural head_dim order, then merge the 4 warps ----
  __syncthreads();
  float* w_o = reinterpret_cast<float*>(smem);   // [4][8][128]
  float* sm_o = w_o + 4 * D8_ROWS * 128;         // [8][128]
  float* w_ml = sm_o + D8_ROWS * 128;            // [4][8][2]
  float* sm_ml = w_ml + 4 * D8_ROWS * 2;         // [8][2]
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int r = 2 * t4 + e;
    if (g == 0) {
      w_ml[(warp * D8_ROWS + r) * 2 + 0] = (m_run[e] == -INFINITY) ? -INFINITY : m_run[e] * p.scale_log2;
      w_ml[(warp * D8_ROWS + r) * 2 + 1] = l_run[e];
    }
    const float off = 1024.f * psT[e];
#pragma unroll
    for (int tl = 0; tl < 8; ++tl) {
      const int call = tl >> 2, ii = tl & 3;
      const float mul = (ii & 1) ? 1.f : 0.0625f;
#pragma unroll
      for (int hm = 0; hm < 2; ++hm) {
        const int d = 32 * (2 * call + hm) + 4 * g + ii;
        w_o[(warp * D8_ROWS + r) * 128 + d] = (oT[tl][hm * 2 + e] - off) * mul + pz_run[e];
      }
    }
  }
  __syncthreads();
  for (int idx = tid; idx < D8_ROWS * 128; idx += I4_THREADS) {
    const int r = idx >> 7, d = idx & 127;
    float mm = -INFINITY;
#pragma unroll
    for (int w = 0; w < 4; ++w) mm = fmaxf(mm, w_ml[(w * D8_ROWS + r) * 2]);
    float acc = 0.f, ll = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float mw = w_ml[(w * D8_ROWS + r) * 2];
      const float f = (mw == -INFINITY) ? 0.f : fast_exp2(mw - mm);
      acc += f * w_o[(w * D8_ROWS + r) * 128 + d];
      ll += f * w_ml[(w * D8_ROWS + r) * 2 + 1];
    }
    sm_o[r * 128 + d] = acc;
    if (d == 0) {
      sm_ml[r * 2] = mm;
      sm_ml[r * 2 + 1] = ll;
    }
  }
  __syncthreads();

  T* outb = reinterpret_cast<T*>(p.out) + (long long)b * p.out_batch_stride;
  float* po_b = nullptr;  // SEQ: part_o[b], part_lse[b]
  float* pl_b = nullptr;
  if constexpr (SEQ) {
    po_b = p.part_o + (long long)b * p.q_len * p.n_q_heads * kHeadDim;
    pl_b = p.part_lse + (long long)b * p.q_len * p.n_q_heads;
  }
  auto store_row_elem = [&](int r, int d, float v0, float v1) {
    const int tok = r / p.group;
    const int hq = kvh * p.group + r % p.group;
    if constexpr (SEQ) {
      if (is_full) {  // the partial of this rank's slice: part_o[b][tok][hq][d]
        *reinterpret_cast<float2*>(po_b + ((long long)tok * p.n_q_heads + hq) * kHeadDim + d) = make_float2(v0, v1);
        return;
      }
    }
    T* dst = outb + ((long long)tok * p.n_q_heads + hq) * kHeadDim + d;
    *reinterpret_cast<uint32_t*>(dst) = MmaOp<T>::pack(v0, v1);
  };
  // SEQ retrieval heads: log2-domain log-sum-exp (scale included) of the row, -inf when no key of the slice is visible
  auto store_row_lse = [&](int r, float m_log2, float l) {
    pl_b[(long long)(r / p.group) * p.n_q_heads + kvh * p.group + r % p.group] = l > 0.f ? m_log2 + log2f(l) : -INFINITY;
  };
  const int nsplit = is_full ? p.splits_full : 1;
  if constexpr (FUSED) {
    if (!is_full) {
      // ---- ring commit (stream_commit_kernel): this CTA was the only reader of the head's ring and has drained its
      // pipeline, so the staged rows of the new tokens may now overwrite their sink / ring slots ----
      for (int w = warp; w < 2 * p.q_len; w += I4_THREADS / 32) {
        const int t = w >> 1;
        const long long pos = p.total + t;
        long long slot;
        if (pos < p.sink) slot = pos;
        else if (t >= p.q_len - p.recent) slot = p.sink + (pos - p.sink) % p.recent;
        else continue;
        const long long srow = (long long)p.stage_off + t;
        uint8_t* base = const_cast<uint8_t*>((w & 1) ? gv : gk);
        *reinterpret_cast<uint16_t*>(base + slot * 64 + lane * 2) = *reinterpret_cast<const uint16_t*>(base + srow * 64 + lane * 2);
        if (lane == 0) {
          __half* sc = const_cast<__half*>((w & 1) ? gvs : gks);
          __half* zp = const_cast<__half*>((w & 1) ? gvz : gkz);
          sc[slot] = sc[srow];
          zp[slot] = zp[srow];
        }
      }
    }
  }
  if (nsplit == 1) {
    for (int idx = tid; idx < rows_total * 64; idx += I4_THREADS) {
      const int r = idx >> 6, d = (idx & 63) * 2;
      const float l = sm_ml[r * 2 + 1];
      const float inv = l > 0.f ? 1.f / l : 0.f;
      store_row_elem(r, d, sm_o[r * 128 + d] * inv, sm_o[r * 128 + d + 1] * inv);
      if constexpr (SEQ) {
        if (is_full && d == 0) store_row_lse(r, sm_ml[r * 2], l);
      }
    }
    return;
  }
  // ---- split-KV publish + hierarchical merge (protocol of attn_mma.cu, 8 rows per item) -----------------------------
  const long long item = RAGGED ? 0 : (long long)b * p.n_full + kvh;  // RAGGED: p.ws is per item
  float* wo = p.ws.ws_o + (item * p.splits_full + split) * (long long)(D8_ROWS * 128);
  float* wml = p.ws.ws_ml + (item * p.splits_full + split) * (long long)(D8_ROWS * 2);
  for (int idx = tid; idx < rows_total * 32; idx += I4_THREADS) {
    const int r = idx >> 5, d4 = (idx & 31) * 4;
    *reinterpret_cast<float4*>(&wo[r * 128 + d4]) = *reinterpret_cast<const float4*>(&sm_o[r * 128 + d4]);
  }
  if (tid < rows_total * 2) wml[tid] = sm_ml[tid];
  DUO_TRACE_STAMP(2);
  // merge scratch: [4][16][128] + [4][16][2] floats = 33 KB of the (drained) 51 KB pipeline ring
  split_kv_finish<D8_ROWS>(p.ws, item, split, p.splits_full, rows_total, reinterpret_cast<float*>(smem),
                           reinterpret_cast<float*>(smem + 32 * 1024), &s_is_last,
                           [&](int r, int d, float v0, float v1, float mm, float ll) {
                             store_row_elem(r, d, v0, v1);
                             if constexpr (SEQ) {
                               if (d == 0) store_row_lse(r, mm, ll);
                             }
                           });
  DUO_TRACE_STAMP(3);
}

// ---------------------------------------------------------------------------------------------
int stage_offset(const duo_layer_desc& d);  // api.cu

// the INT4 cache: packed codes, fp16 scale / zero rows, staging offset and capacities
static void fill_int4_cache(I4Params& p, const duo_layer_desc& d) {
  p.stage_off = stage_offset(d);
  p.full_cap = d.full_cap;
  p.ring_slots = (long long)p.stage_off + d.stage_cap;
  p.full_k = (const uint8_t*)d.full_k;
  p.full_v = (const uint8_t*)d.full_v;
  p.ring_k = (const uint8_t*)d.ring_k;
  p.ring_v = (const uint8_t*)d.ring_v;
  p.fks = (const __half*)d.full_k_scale;
  p.fkz = (const __half*)d.full_k_zero;
  p.fvs = (const __half*)d.full_v_scale;
  p.fvz = (const __half*)d.full_v_zero;
  p.rks = (const __half*)d.ring_k_scale;
  p.rkz = (const __half*)d.ring_k_zero;
  p.rvs = (const __half*)d.ring_v_scale;
  p.rvz = (const __half*)d.ring_v_zero;
}

template <int KEY_WARPS, typename T>
static int launch_i4(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                     int q_len, float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  constexpr int ROWS = 16 * (4 / KEY_WARPS);
  constexpr int I4_TILE = I4Cfg<KEY_WARPS>::TILE;
  I4Params p{};
  fill_common_params(p, d, *st, q, q_row_stride, out, q_len, scale);
  fill_int4_cache(p, d);
  p.n_rb = (d.group * q_len + ROWS - 1) / ROWS;

  // ~2 CTAs per SM, >= 8 tiles per split: 1024 keys with the 128-key tile, 512 with the 64-key tile
  const int full_ctas = d.batch * d.n_full * p.n_rb;
  const SplitPlan sp = plan_splits(st->full_len + q_len, 2 * sm_count_current_device(), full_ctas,
                                   d.batch * d.n_stream * p.n_rb, I4_TILE, 8 * I4_TILE);
  p.splits_full = sp.splits;
  p.keys_per_split = (int)sp.keys_per_split;
  if (sp.splits > 1)
    if (int rc = split_ws_carve(p.ws, split_ws_layout(full_ctas, sp.splits, ROWS), workspace, workspace_bytes,
                                "duo_attention(int4)"))
      return rc;
  const int grid_x = d.n_full * p.n_rb * sp.splits + d.n_stream * p.n_rb;
  if (grid_x == 0) return DUO_OK;
  auto kern = duo_attn_int4_kernel<KEY_WARPS, T>;
  static unsigned long long attr_mask = 0;
  if (int rc = ensure_dyn_smem(kern, I4_SMEM_BYTES, &attr_mask)) return rc;
  kern<<<dim3(grid_x, d.batch), I4_THREADS, I4_SMEM_BYTES, stream>>>(p);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

template <bool FUSED, typename T, bool RAGGED = false, bool POOLED = false, bool SEQ = false>
static int launch_dec8_kernel(dim3 grid, const I4Params& p, cudaStream_t stream) {
  if (grid.x == 0) return DUO_OK;
  auto kern = duo_attn_int4_dec8_kernel<FUSED, T, RAGGED, POOLED, SEQ>;
  static unsigned long long attr_mask = 0;  // per kernel instantiation, one bit per device
  // four CTAs of 51 KB per SM: also ask for the full smem carve-out
  if (int rc = ensure_dyn_smem(kern, D8_SMEM_BYTES, &attr_mask, true)) return rc;
  kern<<<grid, I4_THREADS, D8_SMEM_BYTES, stream>>>(p);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

struct SeqPartials {  // SEQ launches: where the retrieval heads' (O, lse) partials go
  float* part_o = nullptr;
  float* part_lse = nullptr;
};

// Launch of duo_attn_int4_dec8_kernel (group * q_len <= 8): 4 CTAs / SM, 8-row split-KV workspace.  FUSED: the whole
// decode step (duo_decode_fused), q points at the raw qkv rows.  SEQ: a sequence-sharded cache (`st` carries the shard
// descriptor); the split plan covers this rank's local rows.
template <bool FUSED, typename T, bool SEQ = false>
static int launch_i4_dec8(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride,
                          void* out, int q_len, float scale, void* workspace, size_t workspace_bytes,
                          cudaStream_t stream, FusedArgs fa = FusedArgs(), SeqPartials sq = SeqPartials()) {
  const duo_layer_desc& d = L->d;
  I4Params p{};
  fill_common_params(p, d, *st, q, q_row_stride, out, q_len, scale);
  fill_int4_cache(p, d);
  if (FUSED) fill_fused_args(p, fa);
  p.n_rb = 1;
  long long nkeys = st->full_len + q_len;
  if (SEQ) {
    p.part_o = sq.part_o;
    p.part_lse = sq.part_lse;
    p.seq_rank = st->seq_rank;
    p.seq_world = st->seq_world;
    p.seq_block = st->seq_block;
    nkeys = seq_local_len(nkeys, st->seq_rank, st->seq_world, st->seq_block);
  }

  // 4 resident CTAs per SM, >= 1024 keys per split
  const SplitPlan sp = plan_splits(nkeys, 4 * sm_count_current_device(), d.batch * d.n_full,
                                   d.batch * d.n_stream, D8_TILE, 8 * D8_TILE);
  p.splits_full = sp.splits;
  p.keys_per_split = (int)sp.keys_per_split;
  if (sp.splits > 1)
    if (int rc = split_ws_carve(p.ws, split_ws_layout((long long)d.batch * d.n_full, sp.splits, D8_ROWS), workspace,
                                workspace_bytes, "duo_attention(int4/dec8)"))
      return rc;
  return launch_dec8_kernel<FUSED, T, false, false, SEQ>(dim3(d.n_full * sp.splits + d.n_stream, d.batch), p, stream);
}

// ---- ragged decode (duo_decode_ragged_int4): launch_i4_dec8's 4 CTAs/SM budget, 8-row partials --------------------
size_t ragged_int4_workspace_bytes(int batch, int n_kv) { return ragged_ws_need(batch, n_kv, 4, D8_ROWS); }

// row_geom != nullptr: the pooled layout (duo_decode_ragged_pooled), same partition and workspace
int launch_decode_ragged_int4(const duo_layer* L, const long long* row_state, const long long* row_geom,
                              const void* qkv, long long row_stride, const void* cos, const void* sin, int rope_mode,
                              void* out, int q_len, float scale, void* workspace, size_t workspace_bytes,
                              cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  duo_cache_state st{};  // every row's occupancy is read from row_state by the kernel
  st.device_state = reinterpret_cast<const int64_t*>(row_state);
  I4Params p{};
  fill_common_params(p, d, st, qkv, row_stride, out, q_len, scale);
  fill_int4_cache(p, d);
  fill_fused_args(p, {cos, sin, rope_mode});
  p.n_rb = 1;
  const RaggedGeom g = ragged_geom(d.batch, d.n_full, d.n_stream, sm_count_current_device(), 4, D8_ROWS);
  p.rg_slots = g.slots;
  p.rg_want = g.want;
  if (d.n_full > 0)
    if (int rc = split_ws_carve(p.ws, g.ws, workspace, workspace_bytes, "duo_decode_ragged_int4")) return rc;
  const dim3 grid(d.n_full * g.slots + d.batch * d.n_stream, 1);
  p.row_geom = row_geom;
  return dispatch_dtype(d.dtype, [&](auto t) {
    return row_geom ? launch_dec8_kernel<true, decltype(t), true, true>(grid, p, stream)
                    : launch_dec8_kernel<true, decltype(t), true>(grid, p, stream);
  });
}

// One decode-sized chunk over an INT4 cache, everything in one launch (duo_decode_fused): RoPE(q, k) + K1 quantisation
// and append of the new K / V + mixed-head attention + ring commit.  `qkv` is the raw fused projection output; it is
// NOT modified.  group * q_len <= 8 (the keys-as-M kernel).  The activation dtype of the layer picks the instantiation.
int launch_decode_fused_int4(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                             const void* cos, const void* sin, int rope_mode, void* out, int q_len, float scale,
                             void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_i4_dec8<true, decltype(t)>(L, st, qkv, row_stride, out, q_len, scale, workspace, workspace_bytes,
                                             stream, {cos, sin, rope_mode});
  });
}

// Sequence-sharded decode over an INT4 cache (duo_attention_seq_int4): q rotated and this rank's rows appended by
// duo_rope_append; retrieval heads attend the rank's slice and write (O, lse) partials, streaming heads their final
// rows of `out`.  group * q_len <= 8.
int launch_attn_int4_seq(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride,
                         void* out, float* part_o, float* part_lse, int q_len, float scale, void* workspace,
                         size_t workspace_bytes, cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_i4_dec8<false, decltype(t), true>(L, st, q, q_row_stride, out, q_len, scale, workspace,
                                                    workspace_bytes, stream, {}, {part_o, part_lse});
  });
}

// duo_decode_fused_seq_int4: launch_decode_fused_int4 for ONE token of a sequence-sharded cache; only the owner of the
// new position appends it, retrieval heads report partials.
int launch_decode_fused_seq_int4(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                                 const void* cos, const void* sin, int rope_mode, void* out, float* part_o,
                                 float* part_lse, float scale, void* workspace, size_t workspace_bytes,
                                 cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_i4_dec8<true, decltype(t), true>(L, st, qkv, row_stride, out, 1, scale, workspace, workspace_bytes,
                                                   stream, {cos, sin, rope_mode}, {part_o, part_lse});
  });
}

#ifdef DUO_TRACE
extern "C" __attribute__((visibility("default"))) int duo_debug_set_trace(void* buf) {
  return cudaMemcpyToSymbol(g_duo_trace, &buf, sizeof(void*)) == cudaSuccess ? 0 : -3;
}
#endif

template <typename T>
static int launch_attn_int4_t(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride,
                              void* out, int q_len, float scale, void* workspace, size_t workspace_bytes,
                              cudaStream_t stream) {
  if (L->d.group * q_len <= D8_ROWS)
    return launch_i4_dec8<false, T>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes, stream);
  if (L->d.group * q_len <= 16)
    return launch_i4<4, T>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes, stream);
  return launch_i4<1, T>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes, stream);
}

int launch_attn_int4(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                     int q_len, float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_attn_int4_t<decltype(t)>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes, stream);
  });
}

}  // namespace duo
