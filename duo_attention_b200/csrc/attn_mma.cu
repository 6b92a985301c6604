// Mixed-head attention, bandwidth ("decode") kernel family.
//
// One launch serves BOTH head classes of a layer (replaces the two flash_attn_func launches +
// torch.cat of duo_attn/patch/llama.py:234-267 / :374-421):
//   * retrieval kv-heads stream the whole head-major KV cache, split along the key axis over
//     enough CTAs to fill every SM (the count is read at run time); partial (m, l, O) go to a workspace and the LAST CTA of a
//     head to arrive merges them in the same launch (no second kernel);
//   * streaming kv-heads read only the valid sink+ring slots plus the staged chunk.
// K/V tiles (64 keys x 128 dims, K and V) are fetched by TMA (cp.async.bulk.tensor, 128B
// swizzle) into a 3-stage mbarrier pipeline; QK^T and PV run on mma.sync m16n8k16 with fp32
// accumulation reading the swizzled tiles through ldmatrix.  The GQA group (and up to a few
// query tokens) is packed into the 16-row MMA M dimension so each K/V byte is read from HBM
// exactly once.  The kernel is HBM-bound by design; the tensor-core prefill kernel for large
// chunks lives in attn_tc.cu.
//
// Variants:  KEY_WARPS=4 -> 16 packed rows per CTA, the 4 warps split the keys of each tile
//                           (decode: rows = group * q_len <= 16)
//            KEY_WARPS=1 -> 64 packed rows per CTA, each warp owns 16 rows (small chunks and the
//                           generic fallback for ragged prefill shapes)
//            SHARE=1/2   -> the two launches of duo_decode_ragged_shared: a shared prefix streamed once for the
//                           packed rows of every row that shares it (64-row variant), then every row's own keys with
//                           the prefix partial folded into the final store (the pooled ragged decode)
//            SHARE=3     -> a chunk of a row that shares a prefix (duo_attention_shared, 64-row variant): retrieval key
//                           j < share_len is row j of the donor's region (map_pk / map_pv), key j >= share_len row
//                           j - share_len of the own region; tiles, partition and masks are those of a plain row
//            SHARE=4/5   -> the two launches of duo_decode_fused_seq_shared (forks of a sequence-sharded prompt): the
//                           donor's local prefix rows streamed once for the packed rows of every fork (the 64-row
//                           no-causal partial, q rotated in registers), then the sequence-sharded fused decode over the
//                           forks' own slices at positions shifted by share_len, the prefix partial folded into the
//                           stored (O, lse) partial
//            SHARE=6     -> a chunk of forks of a sequence-sharded prompt (duo_prefill_seq_shared, 64-row variant):
//                           the shard mode of duo_prefill_seq, with the slice's local rows [0, share_len) read from the
//                           batch-1 donor and row j >= share_len from own row j - share_len; the one tile across
//                           share_len (a multiple of 8) goes in 8-row pieces (map_pk8 / map_pv8, map_fk8 / map_fv8)
#include <type_traits>

#include "duo_common.cuh"

namespace duo {

constexpr int TILE = 64;                             // keys per pipeline stage
constexpr int STAGES = 3;
constexpr int KV_BOX_BYTES = TILE * 128;             // one 64-wide half of a K or V tile
constexpr int STAGE_BYTES = 4 * KV_BOX_BYTES;        // K lo, K hi, V lo, V hi = 32 KB
constexpr int ATTN_THREADS = 128;

struct AttnParams {
  const void* q;
  void* out;
  long long q_tok_stride;    // elements
  long long q_batch_stride;  // elements
  long long out_batch_stride;
  int q_len, n_q_heads, group, n_full, n_stream, batch;
  int sink, recent, W;
  long long full_len, total, lo;
  const long long* dstate;   // optional device copy of {full_len,total,lo} (CUDA-graph replay)
  float scale_log2;
  int splits_full;       // key splits for retrieval heads
  int keys_per_split;    // multiple of TILE
  int n_rb;              // row blocks per kv head
  int cache_scan;        // streaming: slots [0, cache_scan) are scanned
  SplitWs ws;            // split-KV partials + arrival counters (duo_common.cuh)
  // partial mode (duo_attention_partial / duo_attention_seq): retrieval heads write the fp32 normalised O + log2-domain
  // log-sum-exp of THIS slice of their cache per (token, q head) instead of `out`.
  //   no_causal = 1 (duo_attention_partial): every query row sees all `full_len` keys; only retrieval heads launched
  //   seq_world > 1 (duo_attention_seq): `full_len` counts GLOBAL tokens, the layer's retrieval cache holds the
  //       block-cyclic slice of rank seq_rank (position p lives on rank (p / seq_block) % seq_world, slice order ==
  //       position order); token t sees the local rows of positions <= full_len + t; streaming heads run normally
  float* part_o;
  float* part_lse;
  int no_causal;
  int seq_rank, seq_world, seq_block;
  // FUSED decode step (duo_decode_fused): `q` points at the RAW fused qkv rows; the kernel rotates q in registers,
  // builds the K/V tile of the new tokens in shared memory (K rotated), appends those rows to the caches (retrieval:
  // rows full_len + t; streaming: sink / ring slots, i.e. the ring commit) and attends them — no rope_append /
  // stream_commit launches and no staging round trip.
  const void* cos;
  const void* sin;
  int rope_mode;
  long long k_off, v_off;  // element offsets of the k / v sections inside a qkv row
  void *full_k, *full_v, *ring_k, *ring_v;
  long long full_cap;
  int ring_slots;
  // RAGGED decode (duo_decode_ragged): `dstate` is the [batch][4] row_state array and every batch row has its own
  // occupancy.  The retrieval CTAs of a kv head are rg_slots grid slots shared by all rows; each CTA derives the
  // batch's key partition from row_state (ragged_keys_per_split) and finds its row and split.  ws.n_groups is the
  // per-item stride of the counter and level-2 regions.  Rows flagged idle in row_state (ragged_idle) take no CTA.
  int rg_slots;
  int rg_want;    // split budget per (row, retrieval head) at equal lengths: the `want` of launch_variant
  int rg_budget;  // the CTA budget rg_want came from: the active rows' want when some rows are idle
  // POOLED ragged decode (duo_decode_ragged_pooled): the retrieval K/V of all rows share one pool of
  // pool_tokens * n_full rows; row b's region starts at pool row first_b * n_full and holds [n_full][cap_b][128].
  // row_geom is the device array [batch][2] = {first_b, cap_b} (tokens), read at kernel start.
  const long long* row_geom;
  // SHARED prefixes (duo_decode_ragged_shared): row_share is the device array [batch][2] = {donor d or -1, P}, read at
  // kernel start; a row with d >= 0 and P > 0 attends the donor's keys [0, P) through the prefix kernel.
  //   SHARE == 1, the prefix kernel (64-row variant over the pool): n_full * rg_slots grid slots; a slot is one split of
  //       [0, P) for one 64-row block of the packed rows of the rows that share {d, P} (see share_prefix_slot), which
  //       report fp32 (O, lse) through part_o / part_lse.  rg_want is the most splits one block may take.  dstate
  //       (row_state) is read for the idle flags only: idle rows are not members (share_rank).
  //   SHARE == 2, the suffix kernel (the pooled ragged decode): row b attends its own keys [P_b, full_len_b) and the new
  //       tokens; a sharer's key j lives at row j - P_b of its region, the donor's at row j.  The final store folds in
  //       the row's prefix partial share_o / share_lse (the prefix kernel's part_o / part_lse).
  const long long* row_share;
  const float* share_o;
  const float* share_lse;
};
// rg_budget fills padding: every other field keeps its offset, so no kernel's parameter layout changes
static_assert(offsetof(AttnParams, row_geom) == offsetof(AttnParams, rg_budget) + 4, "AttnParams layout");

// shared-memory scratch of the prefix kernel: the group tables in pipeline stage 2 (not written before the first
// tile), and the member rows of the item behind the merge buffers once the tiles are consumed
constexpr int SHARE_SCRATCH = 2 * STAGE_BYTES;
static_assert(kSharePrefixTile == TILE, "share_prefix_slot plans in 64-key tiles");
constexpr int SHARE_TAB = 88 * 1024;

// rope8<T> (RoPE of 8 head_dim elements and their +64 partners): duo_common.cuh

// same for two packed elements (d, d+1) and their partners (d+64, d+65): the Q fragments of the decode kernel
template <typename T>
__device__ __forceinline__ void rope2(uint32_t& lo2, uint32_t& hi2, const void* cos, const void* sin, int mode, int tok,
                                      int d) {
  T* xl = reinterpret_cast<T*>(&lo2);
  T* xh = reinterpret_cast<T*>(&hi2);
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float a = RopeCvt<T>::to_f(xl[e]), bb = RopeCvt<T>::to_f(xh[e]);
    float ol, oh;
    if (mode == DUO_ROPE_HF) {
      const T* ct = reinterpret_cast<const T*>(cos) + (long long)tok * kHeadDim;
      const T* st = reinterpret_cast<const T*>(sin) + (long long)tok * kHeadDim;
      ol = rope_hf<T>(a, -bb, RopeCvt<T>::to_f(ct[d + e]), RopeCvt<T>::to_f(st[d + e]));
      oh = rope_hf<T>(bb, a, RopeCvt<T>::to_f(ct[d + 64 + e]), RopeCvt<T>::to_f(st[d + 64 + e]));
    } else {
      const float* ct = reinterpret_cast<const float*>(cos) + (long long)tok * kHeadDim;
      const float* st = reinterpret_cast<const float*>(sin) + (long long)tok * kHeadDim;
      ol = rope_f32(a, -bb, ct[d + e], st[d + e]);
      oh = rope_f32(bb, a, ct[d + 64 + e], st[d + 64 + e]);
    }
    xl[e] = RopeCvt<T>::from_f(ol);
    xh[e] = RopeCvt<T>::from_f(oh);
  }
}

// Debug build only (`make trace`, -DDUO_TRACE): per-CTA %globaltimer stamps
#ifdef DUO_TRACE
__device__ unsigned long long* g_duo_trace_mma = nullptr;
__device__ __forceinline__ void trace_stamp_mma(int slot) {
  if (threadIdx.x == 0 && g_duo_trace_mma) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_duo_trace_mma[((long long)blockIdx.y * gridDim.x + blockIdx.x) * 4 + slot] = t;
  }
}
#define DUO_TRACE_MMA(slot) trace_stamp_mma(slot)
#else
#define DUO_TRACE_MMA(slot)
#endif

// (the SHARE == 3 and SHARE == 6 parameters follow the others, so the parameter offsets of every instantiation are the
// same)
template <typename T, int KEY_WARPS, bool FUSED, bool RAGGED = false, bool POOLED = false, int SHARE = 0>
__global__ void __launch_bounds__(ATTN_THREADS, 2)
duo_attn_mma_kernel(const __grid_constant__ CUtensorMap map_fk, const __grid_constant__ CUtensorMap map_fv,
                    const __grid_constant__ CUtensorMap map_rk, const __grid_constant__ CUtensorMap map_rv,
                    const AttnParams pin, const __grid_constant__ CUtensorMap map_pk,
                    const __grid_constant__ CUtensorMap map_pv, const long long share_len,
                    const __grid_constant__ CUtensorMap map_pk8, const __grid_constant__ CUtensorMap map_pv8,
                    const __grid_constant__ CUtensorMap map_fk8, const __grid_constant__ CUtensorMap map_fv8) {
  static_assert(!RAGGED || (FUSED && KEY_WARPS == 4), "the ragged variant is the fused decode kernel");
  static_assert(!POOLED || RAGGED || SHARE == 1, "the pooled layout is a ragged decode layout");
  static_assert(SHARE != 1 || (KEY_WARPS == 1 && !FUSED && !RAGGED && POOLED), "the prefix kernel: 64 rows, pool");
  static_assert(SHARE != 2 || POOLED, "the suffix kernel is the pooled ragged decode");
  static_assert(SHARE != 3 || (KEY_WARPS == 1 && !FUSED && !POOLED), "a sharer's chunk: 64 rows, batch-1 layers");
  static_assert(SHARE != 4 || (KEY_WARPS == 1 && !FUSED && !RAGGED && !POOLED), "the fork prefix: 64 rows, batch 1");
  static_assert(SHARE != 5 || (KEY_WARPS == 4 && FUSED && !RAGGED && !POOLED), "the fork suffix: the fused decode");
  static_assert(SHARE != 6 || (KEY_WARPS == 1 && !FUSED && !RAGGED && !POOLED), "a fork chunk: 64 rows, batch layers");
  DUO_TRACE_MMA(0);
  AttnParams p = pin;
  // (SHARE == 1 reads dstate, the row_state array, for the idle flags only)
  if (!RAGGED && SHARE != 1 && pin.dstate) {  // occupancy lives in device memory: recompute everything that depends on it
    p.full_len = pin.dstate[0];
    if constexpr (SHARE == 5) p.full_len -= share_len;  // the own slices hold positions p - share_len
    p.total = pin.dstate[1];
    p.lo = pin.dstate[2];
    const long long nk = p.seq_world > 1
                             ? seq_local_len(p.full_len + (FUSED ? 0 : p.q_len), p.seq_rank, p.seq_world, p.seq_block)
                             : p.full_len + (FUSED ? 0 : p.q_len);
    p.keys_per_split = (int)split_keys(nk, p.splits_full, TILE);
    p.cache_scan = (int)(p.total < p.W ? p.total : p.W);
  }
  constexpr int ROW_WARPS = 4 / KEY_WARPS;
  constexpr int ROWS = 16 * ROW_WARPS;
  constexpr int KPW = TILE / KEY_WARPS;  // keys per warp per tile
  constexpr int NT = KPW / 8;            // S n-tiles per warp
  using Op = MmaOp<T>;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[STAGES];
  __shared__ int s_is_last;
  __shared__ float s_wmax[2][4][16];  // per-tile row maxima of the 4 key-warps (short contexts only)

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  int b = blockIdx.y;

  // ---- decode the work item ------------------------------------------------------------------
  const int n_full_items = p.n_full * p.n_rb * p.splits_full;
  int kvh, rb, split;
  bool is_full;
  long long key0 = 0, shift = 0;  // SHARE == 2: first own key of the row, and the region row of key j is j - shift
  int share_lead = -1, my_lead = -1, my_rank = 0, share_rows = 0;  // SHARE == 1
  if constexpr (SHARE == 1) {
    const long long* rsh = pin.row_share;
    int* s_lead = reinterpret_cast<int*>(smem + SHARE_SCRATCH);
    int* s_cnt = s_lead + 64;
    int* s_mem = s_lead + 128;
    long long* s_it = reinterpret_cast<long long*>(s_lead + 192);
    if (tid < p.batch) {
      int cnt;
      share_rank(rsh, pin.dstate, p.batch, tid, my_lead, my_rank, cnt);
      s_lead[tid] = my_lead;
      s_cnt[tid] = cnt;
    }
    __syncthreads();
    if (tid == 0)
      share_prefix_slot(rsh, s_lead, s_cnt, p.batch, p.group * p.q_len, p.rg_slots, p.rg_want, blockIdx.x % p.rg_slots,
                        s_it);
    __syncthreads();
    share_lead = (int)s_it[0];
    if (share_lead < 0) return;  // idle slot
    kvh = blockIdx.x / p.rg_slots;
    is_full = true;
    b = (int)rsh[2 * share_lead];  // the donor: its region holds the keys
    p.full_len = rsh[2 * share_lead + 1];
    rb = (int)s_it[1];
    split = (int)s_it[2];
    p.splits_full = (int)s_it[3];
    p.keys_per_split = (int)s_it[4];
    share_rows = (int)s_it[7] * p.group * p.q_len;
    RaggedSlot s;
    s.b = (int)s_it[6];
    s.split = split;
    s.splits = p.splits_full;
    s.slot_base = s_it[5];
    ragged_ws_slice<ROWS>(p.ws, s.b, kvh, p.n_full, p.rg_slots, s);
    if (tid < p.batch && my_lead == share_lead) s_mem[my_rank] = tid;
    __syncthreads();
  } else if constexpr (RAGGED) {
    // grid: n_full * rg_slots retrieval slots (kv-head major), then batch * n_stream streaming CTAs; n_rb == 1
    const long long* rs = pin.dstate;
    rb = 0;
    split = 0;
    const int x = blockIdx.x, n_fslots = p.n_full * p.rg_slots;
    is_full = x < n_fslots;
    if (is_full) {
      // the new tokens are an extra tile (not cache keys): row b's key range is its full_len cached keys
      if constexpr (SHARE == 2) {  // the partition is over the keys the launch reads: a row's shared prefix excluded
        auto own_len = [&](int r) { return rs[4 * r] - share_keys(pin.row_share, r); };
        const long long kps = ragged_batch_kps_of(own_len, rs, p, TILE, 4 * TILE);
        kvh = x / p.rg_slots;
        const RaggedSlot s = ragged_slot_of(own_len, rs, p.batch, kps, x % p.rg_slots);
        b = s.b;
        if (b == p.batch) return;  // idle slot
        split = s.split;
        p.keys_per_split = (int)kps;
        p.splits_full = s.splits;
        ragged_ws_slice<16>(p.ws, b, kvh, p.n_full, p.rg_slots, s);
      } else {
        const long long kps = ragged_batch_kps(rs, p, 0, TILE, 4 * TILE);
        kvh = x / p.rg_slots;
        const RaggedSlot s = ragged_slot(rs, p.batch, 0, kps, x % p.rg_slots);
        b = s.b;
        if (b == p.batch) return;  // idle slot
        split = s.split;
        p.keys_per_split = (int)kps;
        p.splits_full = s.splits;
        ragged_ws_slice<16>(p.ws, b, kvh, p.n_full, p.rg_slots, s);
      }
    } else {
      const int y = x - n_fslots;
      b = y / p.n_stream;
      kvh = p.n_full + y % p.n_stream;
      if (ragged_idle(rs, b)) return;  // an idle row's streaming heads: no load, no ring commit, no store
    }
    p.full_len = rs[4 * b];
    p.total = rs[4 * b + 1];
    p.lo = rs[4 * b + 2];
    p.cache_scan = (int)(p.total < p.W ? p.total : p.W);
    if constexpr (SHARE == 2) {
      key0 = share_keys(pin.row_share, b);
      shift = pin.row_share[2 * b] != b ? key0 : 0;
    }
    // per-row RoPE tables [batch][q_len][128]
    const long long tab = (long long)b * p.q_len * kHeadDim * (p.rope_mode == DUO_ROPE_HF ? (long long)sizeof(T) : 4);
    p.cos = reinterpret_cast<const uint8_t*>(p.cos) + tab;
    p.sin = reinterpret_cast<const uint8_t*>(p.sin) + tab;
  } else if ((int)blockIdx.x < n_full_items) {
    is_full = true;
    int x = blockIdx.x;
    split = x % p.splits_full;
    x /= p.splits_full;
    rb = p.n_rb - 1 - (x % p.n_rb);  // heavy (late) row blocks first
    kvh = x / p.n_rb;
  } else {
    is_full = false;
    int x = blockIdx.x - n_full_items;
    rb = p.n_rb - 1 - (x % p.n_rb);
    kvh = p.n_full + x / p.n_rb;
    split = 0;
  }
  const int rows_total = SHARE == 1 ? share_rows : p.group * p.q_len;
  const int row0 = rb * ROWS;
  const int rows_here = min(ROWS, rows_total - row0);
  const int tok_max = (row0 + rows_here - 1) / p.group;

  // key segments [a0,a1) (cache) and [b0,b1) (staged chunk, streaming heads only)
  long long a0, a1, b0 = 0, b1 = 0;
  // number of keys (of this CTA's key index space) visible to token t: key j is visible  <=>  j < vis_count(t)
  auto vis_count = [&](int t) -> long long {
    if (!is_full) return (long long)p.W + t + 1;
    if (p.no_causal) return p.full_len;
    if (p.seq_world > 1) return seq_local_len(p.full_len + t + 1, p.seq_rank, p.seq_world, p.seq_block);
    return p.full_len + t + 1;
  };
  // FUSED: the new tokens' K/V are not in the caches yet; they form one extra tile built in shared memory, processed
  // after the TMA tiles by the CTA that owns the end of the key range (streaming heads: their only CTA)
  bool has_new = false;
  long long new_base = 0;  // key index of the first new token in this CTA's key index space
  if (is_full) {
    // cached rows of this rank's slice (all of them when the cache is not sequence-sharded)
    const long long cached = p.seq_world > 1 ? seq_local_len(p.full_len, p.seq_rank, p.seq_world, p.seq_block) : p.full_len;
    const long long nkeys = FUSED ? cached : vis_count(tok_max);
    a0 = (long long)split * p.keys_per_split;
    if constexpr (SHARE == 2) a0 += key0;
    a1 = min(nkeys, a0 + (long long)p.keys_per_split);
    if (a1 < a0) a1 = a0;
    has_new = FUSED && (split == p.splits_full - 1);
    if (FUSED && p.seq_world > 1)  // one new token (q_len == 1): only its owner appends and attends it
      has_new = has_new && ((int)((p.full_len / p.seq_block) % p.seq_world) == p.seq_rank);
    new_base = cached;
  } else {
    a0 = 0;
    a1 = p.cache_scan;
    b0 = p.W;
    b1 = FUSED ? b0 : (long long)p.W + tok_max + 1;
    has_new = FUSED;
    new_base = p.W;
  }
  const int nA = (int)((a1 - a0 + TILE - 1) / TILE);
  const int nB = (int)((b1 - b0 + TILE - 1) / TILE);
  const int n_tiles = nA + nB;                       // tiles fetched by TMA
  const int n_iter = n_tiles + (has_new ? 1 : 0);    // + the tile of the new tokens
  const CUtensorMap* mk = is_full ? &map_fk : &map_rk;
  const CUtensorMap* mv = is_full ? &map_fv : &map_rv;
  // POOLED: the retrieval maps span the pool {128, pool_tokens * n_full, 1}; key j of this head is pool row
  // first_b * n_full + kvh * cap_b + j (an int: duo_layer_create_pooled bounds the pool rows)
  int pool_row0 = 0;
  if constexpr (POOLED) {
    if (is_full) pool_row0 = (int)(pin.row_geom[2 * b] * p.n_full + kvh * pin.row_geom[2 * b + 1]);
    if constexpr (SHARE == 2) {
      if (is_full) pool_row0 -= (int)shift;  // a sharer's key j at region row j - P
    }
  }
  const int head_coord = (POOLED && is_full) ? 0 : is_full ? (b * p.n_full + kvh) : (b * p.n_stream + (kvh - p.n_full));

  if (tid == 0) {
    prefetch_tmap(mk);
    prefetch_tmap(mv);
    if constexpr (SHARE == 3 || SHARE == 6) {
      if (is_full) {
        prefetch_tmap(&map_pk);
        prefetch_tmap(&map_pv);
      }
    }
    for (int s = 0; s < STAGES; ++s) mbar_init(&full_bar[s], 1);
    fence_barrier_init();
  }
  __syncthreads();

  auto tile_start = [&](int i) -> long long { return i < nA ? a0 + (long long)i * TILE : b0 + (long long)(i - nA) * TILE; };
  auto issue = [&](int i) {
    const int s = i % STAGES;
    uint8_t* dst = smem + s * STAGE_BYTES;
    const int j0 = (int)tile_start(i) + (POOLED ? pool_row0 : 0);
    if constexpr (SHARE == 3) {  // the donor's rows below share_len, the own region's above (its row j0 - share_len)
      const bool pre = is_full && j0 < share_len;
      const CUtensorMap* tk = pre ? &map_pk : mk;
      const CUtensorMap* tv = pre ? &map_pv : mv;
      const int r0 = (int)(is_full && !pre ? j0 - share_len : j0);
      mbar_expect_tx(&full_bar[s], STAGE_BYTES);
      tma_load_3d(dst, tk, &full_bar[s], 0, r0, head_coord);
      tma_load_3d(dst + KV_BOX_BYTES, tk, &full_bar[s], 64, r0, head_coord);
      tma_load_3d(dst + 2 * KV_BOX_BYTES, tv, &full_bar[s], 0, r0, head_coord);
      tma_load_3d(dst + 3 * KV_BOX_BYTES, tv, &full_bar[s], 64, r0, head_coord);
      return;
    }
    if constexpr (SHARE == 6) {  // the donor's local rows below share_len (head kvh), the own slice's above
      if (is_full) {
        mbar_expect_tx(&full_bar[s], STAGE_BYTES);
        tma_fork_operand<TILE>(dst, KV_BOX_BYTES, &map_pk, mk, &map_pk8, &map_fk8, &full_bar[s], j0, share_len, kvh,
                               head_coord);
        tma_fork_operand<TILE>(dst + 2 * KV_BOX_BYTES, KV_BOX_BYTES, &map_pv, mv, &map_pv8, &map_fv8, &full_bar[s], j0,
                               share_len, kvh, head_coord);
        return;
      }
    }
    mbar_expect_tx(&full_bar[s], STAGE_BYTES);
    tma_load_3d(dst, mk, &full_bar[s], 0, j0, head_coord);
    tma_load_3d(dst + KV_BOX_BYTES, mk, &full_bar[s], 64, j0, head_coord);
    tma_load_3d(dst + 2 * KV_BOX_BYTES, mv, &full_bar[s], 0, j0, head_coord);
    tma_load_3d(dst + 3 * KV_BOX_BYTES, mv, &full_bar[s], 64, j0, head_coord);
  };
  if (tid == 0) {
    for (int i = 0; i < STAGES - 1 && i < n_tiles; ++i) issue(i);
  }

  // ---- Q fragments (registers, loaded once) -----------------------------------------------------
  const int wrow = (KEY_WARPS == 1) ? warp * 16 : 0;  // first packed row of this warp inside the CTA
  const int wkey = (KEY_WARPS == 1) ? 0 : warp * KPW; // first key of this warp inside a tile
  uint32_t qa[8][4];
  int tok_r[2];
  if constexpr (SHARE == 1) {
    // packed row R is token t of member R / (group * q_len) of the group, i.e. token member_row * q_len + t of the
    // batch, of q and of the per-row RoPE tables alike; q is rotated as the fused decode rotates it
    const int* s_mem = reinterpret_cast<const int*>(smem + SHARE_SCRATCH) + 128;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int R = row0 + wrow + g + hf * 8;
      const bool ok = R < rows_total;
      const int tok = ok ? s_mem[R / p.group / p.q_len] * p.q_len + R / p.group % p.q_len : 0;
      const int hq = kvh * p.group + (ok ? R % p.group : 0);
      tok_r[hf] = ok ? tok : -1;
      const T* src = reinterpret_cast<const T*>(p.q) + (long long)tok * p.q_tok_stride + (long long)hq * kHeadDim;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        qa[kk][hf] = ok ? *reinterpret_cast<const uint32_t*>(src + kk * 16 + 2 * t4) : 0u;
        qa[kk][hf + 2] = ok ? *reinterpret_cast<const uint32_t*>(src + kk * 16 + 8 + 2 * t4) : 0u;
      }
      if (ok && p.rope_mode != DUO_ROPE_NONE) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
          for (int half = 0; half < 2; ++half)
            rope2<T>(qa[kk][hf + 2 * half], qa[kk + 4][hf + 2 * half], p.cos, p.sin, p.rope_mode, tok,
                     kk * 16 + half * 8 + 2 * t4);
        }
      }
    }
  } else {
    const T* qb = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_batch_stride;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int R = row0 + wrow + g + hf * 8;
      const bool ok = R < rows_total;
      const int tok = ok ? R / p.group : 0;
      const int hq = kvh * p.group + (ok ? R % p.group : 0);
      tok_r[hf] = ok ? tok : -1;
      const T* src = qb + (long long)tok * p.q_tok_stride + (long long)hq * kHeadDim;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        uint32_t v0 = 0, v1 = 0;
        if (ok) {
          v0 = *reinterpret_cast<const uint32_t*>(src + kk * 16 + 2 * t4);
          v1 = *reinterpret_cast<const uint32_t*>(src + kk * 16 + 8 + 2 * t4);
        }
        qa[kk][hf] = v0;
        qa[kk][hf + 2] = v1;
      }
      if constexpr (FUSED) {
        if (ok && p.rope_mode != DUO_ROPE_NONE) {  // partner of head_dim d is d + 64: k-step kk pairs with kk + 4
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int d = kk * 16 + half * 8 + 2 * t4;
              rope2<T>(qa[kk][hf + 2 * half], qa[kk + 4][hf + 2 * half], p.cos, p.sin, p.rope_mode, tok, d);
            }
          }
        }
      } else if constexpr (SHARE == 4) {
        // the "tokens" are the forks' rows, all at the one new position: every row reads table row 0
        if (ok && p.rope_mode != DUO_ROPE_NONE) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int half = 0; half < 2; ++half)
              rope2<T>(qa[kk][hf + 2 * half], qa[kk + 4][hf + 2 * half], p.cos, p.sin, p.rope_mode, 0,
                       kk * 16 + half * 8 + 2 * t4);
          }
        }
      }
    }
  }

  const long long lim_r[2] = {tok_r[0] >= 0 ? vis_count(tok_r[0]) : 0, tok_r[1] >= 0 ? vis_count(tok_r[1]) : 0};
  const long long lim_min = vis_count((row0 + wrow) / p.group);  // smallest limit among this warp's rows

  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};

  // per-lane ldmatrix address components
  const int lrow = lane & 7;
  const int lmat = lane >> 3;  // 0..3

  for (int i = 0; i < n_iter; ++i) {
    __syncthreads();  // everyone is done with tile i-1 -> its stage may be refilled
    uint32_t sK;
    long long j0, jend;
    if (!FUSED || i < n_tiles) {
      if (tid == 0 && i + STAGES - 1 < n_tiles) issue(i + STAGES - 1);
      const int s = i % STAGES;
      mbar_wait(&full_bar[s], (i / STAGES) & 1);
      sK = smem_u32(smem + s * STAGE_BYTES);
      j0 = tile_start(i);
      jend = (i < nA) ? a1 : b1;
    } else {
      // ---- the new tokens: RoPE(K), append to the caches, build their K/V tile in stage 0 (every TMA tile has been
      // consumed: all stages are free, and for streaming heads the ring has been read, so its slots may be rewritten)
      uint8_t* st0 = smem;
      for (int x = tid; x < STAGE_BYTES / 16; x += ATTN_THREADS) reinterpret_cast<uint4*>(st0)[x] = make_uint4(0, 0, 0, 0);
      __syncthreads();
      const T* rows = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_batch_stride;
      // destination row of new token r in the cache, or -1 if it is not kept (streaming: neither sink nor recent)
      auto dst_row = [&](int r) -> long long {
        if (is_full)  // (local) row of position full_len + r
          return (POOLED ? (long long)pool_row0 : ((long long)b * p.n_full + kvh) * p.full_cap) + new_base + r;
        const long long pos = p.total + r;
        long long slot;
        if (pos < p.sink) slot = pos;
        else if (r >= p.q_len - p.recent) slot = p.sink + (pos - p.sink) % p.recent;
        else return -1;
        return ((long long)b * p.n_stream + (kvh - p.n_full)) * p.ring_slots + slot;
      };
      T* gk = reinterpret_cast<T*>(is_full ? p.full_k : p.ring_k);
      T* gv = reinterpret_cast<T*>(is_full ? p.full_v : p.ring_v);
      for (int w = tid; w < p.q_len * 8; w += ATTN_THREADS) {  // K: (row, 8-element chunk c < 8 and its partner c + 8)
        const int r = w >> 3, c = w & 7;
        const T* src = rows + (long long)r * p.q_tok_stride + p.k_off + (long long)kvh * kHeadDim;
        uint4 lo = *reinterpret_cast<const uint4*>(src + c * 8);
        uint4 hi = *reinterpret_cast<const uint4*>(src + 64 + c * 8);
        if (p.rope_mode != DUO_ROPE_NONE) rope8<T>(lo, hi, p.cos, p.sin, p.rope_mode, r, c * 8);
        const uint32_t off = r * 128 + ((c ^ (r & 7)) << 4);
        *reinterpret_cast<uint4*>(st0 + off) = lo;
        *reinterpret_cast<uint4*>(st0 + KV_BOX_BYTES + off) = hi;
        const long long dr = dst_row(r);
        if (dr >= 0) {
          *reinterpret_cast<uint4*>(gk + dr * kHeadDim + c * 8) = lo;
          *reinterpret_cast<uint4*>(gk + dr * kHeadDim + 64 + c * 8) = hi;
        }
      }
      for (int w = tid; w < p.q_len * 16; w += ATTN_THREADS) {  // V: plain copy
        const int r = w >> 4, c = w & 15;
        const T* src = rows + (long long)r * p.q_tok_stride + p.v_off + (long long)kvh * kHeadDim;
        const uint4 v = *reinterpret_cast<const uint4*>(src + c * 8);
        *reinterpret_cast<uint4*>(st0 + (2 + (c >> 3)) * KV_BOX_BYTES + r * 128 + (((c & 7) ^ (r & 7)) << 4)) = v;
        const long long dr = dst_row(r);
        if (dr >= 0) *reinterpret_cast<uint4*>(gv + dr * kHeadDim + c * 8) = v;
      }
      __syncthreads();
      sK = smem_u32(st0);
      j0 = new_base;
      jend = new_base + p.q_len;
    }
    const uint32_t sV = sK + 2 * KV_BOX_BYTES;

    // ---- S = Q K^T ------------------------------------------------------------------------------
    float sc[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int pr = 0; pr < NT / 2; ++pr) {
        const int krow = wkey + pr * 16 + (lmat >> 1) * 8 + lrow;
        const int cc = kk * 2 + (lmat & 1);  // 16-byte chunk index 0..15 along head_dim
        const uint32_t addr = sK + (cc >> 3) * KV_BOX_BYTES + krow * 128 + (((cc & 7) ^ (krow & 7)) << 4);
        uint32_t r0, r1, r2, r3;
        ldsm_x4(r0, r1, r2, r3, addr);
        Op::run(sc[2 * pr], qa[kk], r0, r1);
        Op::run(sc[2 * pr + 1], qa[kk], r2, r3);
      }
    }

    // ---- mask + online softmax ----------------------------------------------------------------
    const long long kfirst = j0 + wkey;
    const bool need_mask = (kfirst + KPW > jend) || (kfirst + KPW > lim_min) ||
                           (!is_full && i < nA);  // rows beyond rows_here hold q == 0 and are never stored
    if (need_mask) {
#pragma unroll
      for (int n = 0; n < NT; ++n) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const long long j = kfirst + n * 8 + 2 * t4 + (e & 1);
          bool vis = (j < jend) && (j < lim_r[e >> 1]);
          if (!is_full && j < p.W) vis = vis && stream_slot_valid((int)j, p.sink, p.recent, p.total, p.lo);
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
    if constexpr (KEY_WARPS == 4) {
      // Short contexts: let the 4 key-warps agree on one row max per tile, so P is rounded against the same
      // reference a single-block kernel (FA2 / the oracle) uses; with only a few dozen keys the independent
      // per-warp references would otherwise be the largest source of bf16 rounding noise.  Long contexts
      // average that noise out and skip the extra barrier.
      if (n_iter <= 8) {
        if (t4 == 0) {
          s_wmax[i & 1][warp][g] = mx[0];
          s_wmax[i & 1][warp][g + 8] = mx[1];
        }
        __syncthreads();
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          mx[0] = fmaxf(mx[0], s_wmax[i & 1][w][g]);
          mx[1] = fmaxf(mx[1], s_wmax[i & 1][w][g + 8]);
        }
      }
    }
    float alpha[2], msc[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const float m_new = fmaxf(m_run[hf], mx[hf]);
      msc[hf] = (m_new == -INFINITY) ? 0.f : m_new * p.scale_log2;
      alpha[hf] = (m_run[hf] == -INFINITY) ? 0.f : fast_exp2(m_run[hf] * p.scale_log2 - msc[hf]);
      m_run[hf] = m_new;
    }
    float rs[2] = {0.f, 0.f};
    uint32_t pa[NT / 2][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const float p0 = fast_exp2(sc[n][0] * p.scale_log2 - msc[0]);
      const float p1 = fast_exp2(sc[n][1] * p.scale_log2 - msc[0]);
      const float p2 = fast_exp2(sc[n][2] * p.scale_log2 - msc[1]);
      const float p3 = fast_exp2(sc[n][3] * p.scale_log2 - msc[1]);
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      // accumulator layout of two adjacent n-tiles == A fragment of one k16 step
      pa[n >> 1][(n & 1) * 2 + 0] = Op::pack(p0, p1);
      pa[n >> 1][(n & 1) * 2 + 1] = Op::pack(p2, p3);
    }
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) l_run[hf] = l_run[hf] * alpha[hf] + rs[hf];
#pragma unroll
    for (int d = 0; d < 16; ++d) {
      o[d][0] *= alpha[0];
      o[d][1] *= alpha[0];
      o[d][2] *= alpha[1];
      o[d][3] *= alpha[1];
    }

    // ---- O += P V -------------------------------------------------------------------------------
#pragma unroll
    for (int k2 = 0; k2 < NT / 2; ++k2) {
#pragma unroll
      for (int q2 = 0; q2 < 8; ++q2) {
        const int krow = wkey + k2 * 16 + (lmat & 1) * 8 + lrow;
        const int cc = q2 * 2 + (lmat >> 1);
        const uint32_t addr = sV + (cc >> 3) * KV_BOX_BYTES + krow * 128 + (((cc & 7) ^ (krow & 7)) << 4);
        uint32_t r0, r1, r2, r3;
        ldsm_x4_trans(r0, r1, r2, r3, addr);
        Op::run(o[2 * q2], pa[k2], r0, r1);
        Op::run(o[2 * q2 + 1], pa[k2], r2, r3);
      }
    }
  }

  DUO_TRACE_MMA(1);
  // row sums live distributed over the 4 lanes of a quad
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 1);
    l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 2);
  }

  // ---- cross-warp merge (KEY_WARPS == 4): every warp holds partials for the same 16 rows ---------
  __syncthreads();  // all TMA tiles consumed -> pipeline smem is free for reuse
  float* sm_o = reinterpret_cast<float*>(smem);                 // [ROWS][128] merged, unnormalised
  float* sm_ml = reinterpret_cast<float*>(smem + 64 * 1024);    // [ROWS][2]   (m in log2 units, l)
  int* s_tab = reinterpret_cast<int*>(smem + SHARE_TAB);         // SHARE == 1: member index -> batch row
  if constexpr (SHARE == 1) {
    if (tid < p.batch && my_lead == share_lead) s_tab[my_rank] = tid;
  }
  if constexpr (KEY_WARPS == 4) {
    float* w_o = reinterpret_cast<float*>(smem) + 16 * 128;     // [4][16][128] behind the merged block
    float* w_ml = sm_ml + 64;                                   // [4][16][2]
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int r = g + hf * 8;
      if (t4 == 0) {
        w_ml[(warp * 16 + r) * 2 + 0] = (m_run[hf] == -INFINITY) ? -INFINITY : m_run[hf] * p.scale_log2;
        w_ml[(warp * 16 + r) * 2 + 1] = l_run[hf];
      }
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        float2 v = make_float2(o[d][hf * 2], o[d][hf * 2 + 1]);
        *reinterpret_cast<float2*>(&w_o[(warp * 16 + r) * 128 + d * 8 + 2 * t4]) = v;
      }
    }
    __syncthreads();
    for (int idx = tid; idx < 16 * 128; idx += ATTN_THREADS) {
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
  } else {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int r = wrow + g + hf * 8;
      if (t4 == 0) {
        sm_ml[r * 2 + 0] = (m_run[hf] == -INFINITY) ? -INFINITY : m_run[hf] * p.scale_log2;
        sm_ml[r * 2 + 1] = l_run[hf];
      }
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        float2 v = make_float2(o[d][hf * 2], o[d][hf * 2 + 1]);
        *reinterpret_cast<float2*>(&sm_o[r * 128 + d * 8 + 2 * t4]) = v;
      }
    }
  }
  __syncthreads();

  T* outb = reinterpret_cast<T*>(p.out) + (long long)b * p.out_batch_stride;
  // SHARE == 1: the (token, q head) row of the partials of packed row R, a member's row of the group
  auto share_row = [&](int R) -> long long {
    const int rpm = p.group * p.q_len, w = R % rpm;
    return ((long long)s_tab[R / rpm] * p.q_len + w / p.group) * p.n_q_heads + kvh * p.group + w % p.group;
  };
  auto store_row_elem = [&](int r, int d, float v0, float v1) {
    const int R = row0 + r;
    if constexpr (SHARE == 1) {
      *reinterpret_cast<float2*>(p.part_o + share_row(R) * kHeadDim + d) = make_float2(v0, v1);
      return;
    }
    const int tok = R / p.group;
    const int hq = kvh * p.group + R % p.group;
    if (p.part_o && is_full) {
      float* dst = p.part_o + (((long long)b * p.q_len + tok) * p.n_q_heads + hq) * kHeadDim + d;
      *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
      return;
    }
    T* dst = outb + ((long long)tok * p.n_q_heads + hq) * kHeadDim + d;
    *reinterpret_cast<uint32_t*>(dst) = Op::pack(v0, v1);
  };
  auto store_row_lse = [&](int r, float m_log2, float l) {  // partial mode only
    const int R = row0 + r;
    if constexpr (SHARE == 1) {
      p.part_lse[share_row(R)] = l > 0.f ? m_log2 + log2f(l) : -INFINITY;
      return;
    }
    p.part_lse[((long long)b * p.q_len + R / p.group) * p.n_q_heads + kvh * p.group + R % p.group] =
        l > 0.f ? m_log2 + log2f(l) : -INFINITY;
  };
  // the final (normalised) value of dims d, d+1 of row r; SHARE == 2 folds in the row's prefix partial first (the
  // online-softmax rule: weights 2^lse_prefix and l * 2^m of the own keys)
  auto store_final = [&](int r, int d, float v0, float v1, float mm, float ll) {
    if constexpr (SHARE == 2) {
      if (is_full && key0 > 0) {
        const int R = row0 + r;
        const long long row = ((long long)b * p.q_len + R / p.group) * p.n_q_heads + kvh * p.group + R % p.group;
        const float lp = p.share_lse[row];
        const float2 op = *reinterpret_cast<const float2*>(p.share_o + row * kHeadDim + d);
        const float M = fmaxf(lp, mm);
        const float ws = mm == -INFINITY ? 0.f : ll * fast_exp2(mm - M);
        const float wp = lp == -INFINITY ? 0.f : fast_exp2(lp - M);
        const float inv = ws + wp > 0.f ? 1.f / (ws + wp) : 0.f;
        v0 = (ws * v0 + wp * op.x) * inv;
        v1 = (ws * v1 + wp * op.y) * inv;
      }
    }
    if constexpr (SHARE == 5) {  // the same rule, and the partial's lse becomes that of prefix and own keys together
      if (is_full) {
        const int R = row0 + r;
        const long long row = ((long long)b * p.q_len + R / p.group) * p.n_q_heads + kvh * p.group + R % p.group;
        const float lp = p.share_lse[row];
        const float2 op = *reinterpret_cast<const float2*>(p.share_o + row * kHeadDim + d);
        const float M = fmaxf(lp, mm);
        const float ws = mm == -INFINITY ? 0.f : ll * fast_exp2(mm - M);
        const float wp = lp == -INFINITY ? 0.f : fast_exp2(lp - M);
        const float inv = ws + wp > 0.f ? 1.f / (ws + wp) : 0.f;
        v0 = (ws * v0 + wp * op.x) * inv;
        v1 = (ws * v1 + wp * op.y) * inv;
        if (d == 0) p.part_lse[row] = ws + wp > 0.f ? M + log2f(ws + wp) : -INFINITY;
      }
    }
    store_row_elem(r, d, v0, v1);
  };

  const int nsplit = is_full ? p.splits_full : 1;
  if (nsplit == 1) {
    for (int idx = tid; idx < rows_here * 64; idx += ATTN_THREADS) {
      const int r = idx >> 6, d = (idx & 63) * 2;
      const float l = sm_ml[r * 2 + 1];
      const float inv = l > 0.f ? 1.f / l : 0.f;
      if constexpr (SHARE == 2 || SHARE == 5)
        store_final(r, d, sm_o[r * 128 + d] * inv, sm_o[r * 128 + d + 1] * inv, sm_ml[r * 2], l);
      else
        store_row_elem(r, d, sm_o[r * 128 + d] * inv, sm_o[r * 128 + d + 1] * inv);
      if (SHARE != 5 && p.part_lse && is_full && d == 0) store_row_lse(r, sm_ml[r * 2], l);
    }
    return;
  }

  // ---- split-KV: publish the partial; group / final merges by the last arrivals (split_kv_finish) ----------------
  // RAGGED, SHARE == 1: p.ws is per item
  const long long item = (RAGGED || SHARE == 1) ? 0 : ((long long)b * p.n_full + kvh) * p.n_rb + rb;
  float* wo = p.ws.ws_o + (item * p.splits_full + split) * (long long)(ROWS * 128);
  float* wml = p.ws.ws_ml + (item * p.splits_full + split) * (long long)(ROWS * 2);
  for (int idx = tid; idx < rows_here * 32; idx += ATTN_THREADS) {
    const int r = idx >> 5, d4 = (idx & 31) * 4;
    *reinterpret_cast<float4*>(&wo[r * 128 + d4]) = *reinterpret_cast<const float4*>(&sm_o[r * 128 + d4]);
  }
  if (tid < rows_here * 2) wml[tid] = sm_ml[tid];
  DUO_TRACE_MMA(2);
  split_kv_finish<ROWS>(p.ws, item, split, p.splits_full, rows_here, reinterpret_cast<float*>(smem),
                        reinterpret_cast<float*>(smem + 80 * 1024), &s_is_last,
                        [&](int r, int d, float v0, float v1, float mm, float ll) {
                          if constexpr (SHARE == 2 || SHARE == 5)
                            store_final(r, d, v0, v1, mm, ll);
                          else
                            store_row_elem(r, d, v0, v1);
                          if (SHARE != 5 && p.part_lse && d == 0) store_row_lse(r, mm, ll);
                        });
  DUO_TRACE_MMA(3);
}

// ---------------------------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------------------------
constexpr int ATTN_SMEM_BYTES = STAGES * STAGE_BYTES + 1024;  // + alignment slack

size_t mma_workspace_bytes(int batch, int n_kv, int group, int max_q_len) {
  // The launchers never create more than ~4 CTAs/SM worth of split partials (items * splits <= budget), each at most
  // 64 rows x (128 + 2) floats, plus one level-2 partial per group of kMergeGroup splits and per item, plus counters.
  const long long max_partials = 4 * 160 + 64;
  const long long rows = (long long)group * max_q_len;
  const long long items = (long long)batch * n_kv * ((rows + 15) / 16);
  const long long l1 = max_partials * 64 * 130 * 4;
  const long long l2 = (max_partials / kMergeGroup + items + 8) * 64 * 130 * 4;
  return (size_t)(kSplitCounterBytes + l1 + l2 + 8192);
}

struct PartialMode {      // how the retrieval heads report (see AttnParams)
  float* part_o = nullptr;
  float* part_lse = nullptr;
  bool no_causal = false;  // duo_attention_partial: plain slice, streaming heads not launched
  const float* share_o = nullptr;    // SHARE == 5: the forks' prefix partials, folded into the stored ones
  const float* share_lse = nullptr;
};
int stage_offset(const duo_layer_desc& d);  // api.cu
int encode_piece_maps(const duo_layer* L, CUtensorMap* k8, CUtensorMap* v8);  // api.cu

// fused decode step: RoPE inputs, and the caches the kernel appends the new rows to
static void fill_fused(AttnParams& p, const duo_layer_desc& d, const FusedArgs& fa) {
  fill_fused_args(p, fa);
  p.full_k = d.full_k;
  p.full_v = d.full_v;
  p.ring_k = d.ring_k;
  p.ring_v = d.ring_v;
  p.full_cap = d.full_cap;
  p.ring_slots = stage_offset(d) + d.stage_cap;
}

// the launch attributes of one instantiation (set once per device)
template <typename T, int KEY_WARPS, bool FUSED, bool RAGGED = false, bool POOLED = false, int SHARE = 0>
static int prepare_mma_kernel() {
  static unsigned long long attr_mask = 0;  // per kernel instantiation, one bit per device
  return ensure_dyn_smem(duo_attn_mma_kernel<T, KEY_WARPS, FUSED, RAGGED, POOLED, SHARE>, ATTN_SMEM_BYTES, &attr_mask);
}

// SHARE == 3 / 6: the first share_len retrieval keys (6: local rows of the slice) are rows of `prefix`; other modes pass
// the own maps in those slots.  SHARE == 6 also takes 8-row-box maps of both, encoded here.
template <typename T, int KEY_WARPS, bool FUSED, bool RAGGED = false, bool POOLED = false, int SHARE = 0>
static int launch_mma_kernel(const duo_layer* L, dim3 grid, const AttnParams& p, cudaStream_t stream,
                             const duo_layer* prefix = nullptr, long long share_len = 0) {
  if (grid.x == 0) return DUO_OK;
  auto kern = duo_attn_mma_kernel<T, KEY_WARPS, FUSED, RAGGED, POOLED, SHARE>;
  if (int rc = prepare_mma_kernel<T, KEY_WARPS, FUSED, RAGGED, POOLED, SHARE>()) return rc;
  const KvMaps m = kv_maps(L, false);
  const KvMaps pm = kv_maps(SHARE == 3 || SHARE == 6 ? prefix : L, false);
  CUtensorMap piece[4] = {*pm.fk, *pm.fv, *m.fk, *m.fv};
  if (SHARE == 6 && L->d.n_full > 0) {
    if (int rc = encode_piece_maps(prefix, &piece[0], &piece[1])) return rc;
    if (int rc = encode_piece_maps(L, &piece[2], &piece[3])) return rc;
  }
  kern<<<grid, ATTN_THREADS, ATTN_SMEM_BYTES, stream>>>(*m.fk, *m.fv, *m.rk, *m.rv, p, *pm.fk, *pm.fv, share_len,
                                                        piece[0], piece[1], piece[2], piece[3]);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

template <typename T, int KEY_WARPS, bool FUSED = false, int SHARE = 0>
static int launch_variant(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride,
                          void* out, int q_len, float scale, void* workspace, size_t workspace_bytes,
                          cudaStream_t stream, PartialMode pm = PartialMode(), FusedArgs fa = FusedArgs(),
                          const duo_layer* prefix = nullptr, long long share_len = 0) {
  const duo_layer_desc& d = L->d;
  constexpr int ROWS = 16 * (4 / KEY_WARPS);
  AttnParams p{};
  fill_common_params(p, d, *st, q, q_row_stride, out, q_len, scale);
  if (FUSED) fill_fused(p, d, fa);
  if (SHARE == 4) fill_fused_args(p, fa);  // q is rotated in registers; nothing is appended
  p.n_rb = (d.group * q_len + ROWS - 1) / ROWS;
  const bool partial = pm.no_causal;  // slice-only launch: no streaming CTAs
  p.part_o = pm.part_o;
  p.part_lse = pm.part_lse;
  p.share_o = pm.share_o;
  p.share_lse = pm.share_lse;
  p.no_causal = pm.no_causal ? 1 : 0;
  p.seq_rank = st->seq_rank;
  p.seq_world = st->seq_world;
  p.seq_block = st->seq_block;

  // split the retrieval heads' keys so that the grid covers ~2 CTAs per SM, >= 256 keys per split
  const long long seen = (partial || FUSED) ? st->full_len : st->full_len + q_len;  // positions the TMA tiles cover
  const long long nkeys = (!partial && st->seq_world > 1) ? seq_local_len(seen, st->seq_rank, st->seq_world, st->seq_block)
                                                          : seen;
  const int full_ctas = d.batch * d.n_full * p.n_rb, stream_ctas = partial ? 0 : d.batch * d.n_stream * p.n_rb;
  const SplitPlan sp = plan_splits(nkeys, 2 * sm_count_current_device(), full_ctas, stream_ctas, TILE, 4 * TILE);
  p.splits_full = sp.splits;
  p.keys_per_split = (int)sp.keys_per_split;
  if (sp.splits > 1)
    if (int rc = split_ws_carve(p.ws, split_ws_layout(full_ctas, sp.splits, ROWS), workspace, workspace_bytes,
                                "duo_attention"))
      return rc;

  const int grid_x = d.n_full * p.n_rb * sp.splits + (partial ? 0 : d.n_stream * p.n_rb);
  return launch_mma_kernel<T, KEY_WARPS, FUSED, false, false, SHARE>(L, dim3(grid_x, d.batch), p, stream, prefix,
                                                                     share_len);
}

int launch_attn_mma(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                    int q_len, float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const bool decode_rows = L->d.group * q_len <= 16;
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    using T = decltype(t);
    return decode_rows ? launch_variant<T, 4>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes, stream)
                       : launch_variant<T, 1>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes, stream);
  });
}

// A chunk of group * q_len > 16 rows of a row whose first share_len retrieval keys are rows of `prefix`
// (duo_attention_shared): the 64-row variant with the plain row's split-KV partition.
int launch_attn_mma_shared(const duo_layer* L, const duo_layer* prefix, long long share_len, const duo_cache_state* st,
                           const void* q, long long q_row_stride, void* out, int q_len, float scale, void* workspace,
                           size_t workspace_bytes, cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_variant<decltype(t), 1, false, 3>(L, st, q, q_row_stride, out, q_len, scale, workspace,
                                                    workspace_bytes, stream, {}, {}, prefix, share_len);
  });
}

// out[tok][h][:] = sum_p w_p o_p / sum_p w_p, w_p = 2^(lse_p - max_p lse_p): the cross-slice step of the online softmax
// (same algebra as the last-CTA split-KV merge, one level up).  Only heads h < heads_used are touched.
template <typename T>
__global__ void __launch_bounds__(128) merge_partials_kernel(const float* __restrict__ o_parts,
                                                             const float* __restrict__ lse_parts, int n_parts,
                                                             long long tokens, int heads_total, int heads_used,
                                                             T* __restrict__ out) {
  const long long tok = blockIdx.x / heads_used;
  const int h = (int)(blockIdx.x % heads_used);
  const long long row = tok * heads_total + h;
  const long long part_rows = tokens * heads_total;
  float mx = -INFINITY;
  for (int q = 0; q < n_parts; ++q) mx = fmaxf(mx, lse_parts[q * part_rows + row]);
  float acc = 0.f, wsum = 0.f;
  for (int q = 0; q < n_parts; ++q) {
    const float l = lse_parts[q * part_rows + row];
    if (l == -INFINITY) continue;
    const float w = fast_exp2(l - mx);
    acc += w * o_parts[(q * part_rows + row) * kHeadDim + threadIdx.x];
    wsum += w;
  }
  const float v = wsum > 0.f ? acc / wsum : 0.f;
  if constexpr (sizeof(T) == 2 && std::is_same<T, __nv_bfloat16>::value)
    out[row * kHeadDim + threadIdx.x] = __float2bfloat16_rn(v);
  else
    out[row * kHeadDim + threadIdx.x] = __float2half_rn(v);
}

int launch_merge_partials(const float* o_parts, const float* lse_parts, int n_parts, long long tokens, int heads_total,
                          int heads_used, void* out, int dtype, cudaStream_t stream) {
  if (tokens == 0 || heads_used == 0) return DUO_OK;
  const unsigned grid = (unsigned)(tokens * heads_used);
  return dispatch_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    merge_partials_kernel<T><<<grid, 128, 0, stream>>>(o_parts, lse_parts, n_parts, tokens, heads_total, heads_used,
                                                       (T*)out);
    DUO_CUDA_TRY(cudaGetLastError());
    return DUO_OK;
  });
}

// Partial attention over the first n_keys rows of every retrieval head (building block of the sequence-sharded
// decode, DESIGN.md section 6): decode-sized q only.
int launch_attn_mma_partial(const duo_layer* L, long long n_keys, const void* q, long long q_row_stride, float* out_o,
                            float* out_lse, int q_len, float scale, void* workspace, size_t workspace_bytes,
                            cudaStream_t stream) {
  duo_cache_state st{};
  st.full_len = n_keys;
  st.lo = L->d.sink;
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_variant<decltype(t), 4>(L, &st, q, q_row_stride, nullptr, q_len, scale, workspace, workspace_bytes,
                                          stream, {out_o, out_lse, true});
  });
}

#ifdef DUO_TRACE
extern "C" __attribute__((visibility("default"))) int duo_debug_set_trace_mma(void* buf) {
  return cudaMemcpyToSymbol(g_duo_trace_mma, &buf, sizeof(void*)) == cudaSuccess ? 0 : -3;
}
#endif

// One decode-sized chunk, everything in one launch (duo_decode_fused): RoPE(q, k) + KV append + mixed-head attention +
// ring commit.  `qkv` is the raw fused projection output; it is NOT modified.
int launch_decode_fused(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                        const void* cos, const void* sin, int rope_mode, void* out, int q_len, float scale,
                        void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_variant<decltype(t), 4, true>(L, st, qkv, row_stride, out, q_len, scale, workspace, workspace_bytes,
                                                stream, {}, {cos, sin, rope_mode});
  });
}

// ---- ragged decode (duo_decode_ragged): launch_variant's ~2 CTAs/SM budget, 16-row partials ---------------------
size_t ragged_workspace_bytes(int batch, int n_kv) { return ragged_ws_need(batch, n_kv, 2, 16); }

// row_geom != nullptr: the pooled layout (duo_decode_ragged_pooled), same partition and workspace
int launch_decode_ragged(const duo_layer* L, const long long* row_state, const long long* row_geom, const void* qkv,
                         long long row_stride, const void* cos, const void* sin, int rope_mode, void* out, int q_len,
                         float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  duo_cache_state st{};  // every row's occupancy is read from row_state by the kernel
  st.device_state = reinterpret_cast<const int64_t*>(row_state);
  AttnParams p{};
  fill_common_params(p, d, st, qkv, row_stride, out, q_len, scale);
  fill_fused(p, d, {cos, sin, rope_mode});
  p.n_rb = 1;
  const RaggedGeom g = ragged_geom(d.batch, d.n_full, d.n_stream, sm_count_current_device(), 2, 16);
  p.rg_slots = g.slots;
  p.rg_want = g.want;
  p.rg_budget = g.budget;
  if (d.n_full > 0)
    if (int rc = split_ws_carve(p.ws, g.ws, workspace, workspace_bytes, "duo_decode_ragged")) return rc;
  const dim3 grid(d.n_full * g.slots + d.batch * d.n_stream, 1);
  p.row_geom = row_geom;
  return dispatch_dtype(d.dtype, [&](auto t) {
    return row_geom ? launch_mma_kernel<decltype(t), 4, true, true, true>(L, grid, p, stream)
                    : launch_mma_kernel<decltype(t), 4, true, true>(L, grid, p, stream);
  });
}

// ---- shared prefixes (duo_decode_ragged_shared) ----------------------------------------------------------------
size_t ragged_shared_workspace_bytes(int batch, int n_kv) {
  const int sms = sm_count_current_device();
  size_t need = 0;
  for (int nf = 1; nf <= n_kv; ++nf) {
    const size_t b = shared_split_bytes(ragged_geom(batch, nf, n_kv - nf, sms, 2, 16), prefix_geom(batch, nf, sms));
    if (b == (size_t)-1) return b;
    need = std::max(need, b);
  }
  const size_t rows = (size_t)batch * DUO_DECODE_MAX_Q * n_kv;  // q_len * n_q_heads = q_len * group * n_kv
  return need + rows * (kHeadDim + 1) * 4;
}

int launch_decode_ragged_shared(const duo_layer* L, const long long* row_state, const long long* row_geom,
                                const long long* row_share, const void* qkv, long long row_stride, const void* cos,
                                const void* sin, int rope_mode, void* out, int q_len, float scale, void* workspace,
                                size_t workspace_bytes, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  const int sms = sm_count_current_device();
  duo_cache_state st{};  // every row's occupancy is read from row_state by the kernels
  st.device_state = reinterpret_cast<const int64_t*>(row_state);
  AttnParams p{};
  fill_common_params(p, d, st, qkv, row_stride, out, q_len, scale);
  fill_fused(p, d, {cos, sin, rope_mode});
  p.n_rb = 1;
  const RaggedGeom g = ragged_geom(d.batch, d.n_full, d.n_stream, sms, 2, 16);
  p.rg_slots = g.slots;
  p.rg_want = g.want;
  p.rg_budget = g.budget;
  p.row_geom = row_geom;
  p.row_share = row_share;
  AttnParams pp = p;  // the prefix launch: retrieval heads only, no occupancy but the shared keys and the idle flags
  const PrefixGeom pg = prefix_geom(d.batch, d.n_full, sms);
  if (d.n_full > 0) {
    const size_t off = shared_split_bytes(g, pg);
    const long long rows = (long long)d.batch * q_len * p.n_q_heads;
    const size_t need = off == (size_t)-1 ? off : off + (size_t)rows * (kHeadDim + 1) * 4;
    if (need == (size_t)-1 || workspace == nullptr || workspace_bytes < need) {
      set_error("duo_decode_ragged_shared: workspace too small (%zu < %zu)", workspace_bytes, need);
      return DUO_EWORKSPACE;
    }
    float* pre_o = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + off);
    float* pre_lse = pre_o + rows * kHeadDim;
    if (int rc = split_ws_carve(p.ws, g.ws, workspace, workspace_bytes, "duo_decode_ragged_shared")) return rc;
    if (int rc = split_ws_carve(pp.ws, pg.ws, workspace, workspace_bytes, "duo_decode_ragged_shared")) return rc;
    p.share_o = pre_o;
    p.share_lse = pre_lse;
    pp.no_causal = 1;
    pp.part_o = pre_o;
    pp.part_lse = pre_lse;
    pp.rg_slots = pg.slots;
    pp.rg_want = pg.max_splits;
  }
  const dim3 grid(d.n_full * g.slots + d.batch * d.n_stream, 1);
  return dispatch_dtype(d.dtype, [&](auto t) {
    using T = decltype(t);
    // both kernels are set up before either is enqueued: a failed call leaves nothing launched
    if (int rc = prepare_mma_kernel<T, 1, false, false, true, 1>()) return rc;
    if (int rc = prepare_mma_kernel<T, 4, true, true, true, 2>()) return rc;
    if (d.n_full > 0)
      if (int rc = launch_mma_kernel<T, 1, false, false, true, 1>(L, dim3(d.n_full * pg.slots, 1), pp, stream)) return rc;
    return launch_mma_kernel<T, 4, true, true, true, 2>(L, grid, p, stream);
  });
}

// duo_decode_fused for a sequence-sharded cache (ONE new token): as launch_decode_fused, retrieval heads report partials.
int launch_decode_fused_seq(const duo_layer* L, const duo_cache_state* st, const void* qkv, long long row_stride,
                            const void* cos, const void* sin, int rope_mode, void* out, float* part_o, float* part_lse,
                            float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_variant<decltype(t), 4, true>(L, st, qkv, row_stride, out, 1, scale, workspace, workspace_bytes, stream,
                                                {part_o, part_lse}, {cos, sin, rope_mode});
  });
}

// ---- forks of a sequence-sharded prompt (duo_decode_fused_seq_shared) --------------------------------------------
// Split-KV bytes of the two launches for any layer of n_kv heads and group <= 16 on this device: they run one after the
// other and share one region (each leaves its counters zeroed).  Splits are bounded by split_want's budget whatever
// the key count, and fewer splits need fewer bytes, so the bound holds at every length.
static size_t seq_shared_split_bytes(int batch, int n_kv) {
  const int budget = 2 * sm_count_current_device();
  size_t need = 0;
  for (int nf = 1; nf <= n_kv; ++nf) {
    for (int group = 1; group <= 16; ++group) {
      const long long pre_items = (long long)nf * ((batch * group + 63) / 64), suf_items = (long long)batch * nf;
      const int pre = std::min(512, split_want(budget, (int)pre_items, 0));
      const int suf = std::min(512, split_want(budget, (int)suf_items, batch * (n_kv - nf)));
      for (const SplitWsLayout& l : {split_ws_layout(pre_items, pre, 64), split_ws_layout(suf_items, suf, 16)}) {
        const size_t b = split_ws_bytes(l);
        if (b == (size_t)-1) return b;
        need = std::max(need, b);
      }
    }
  }
  return (need + 255) / 256 * 256;
}

// the split region, then the prefix partials: [batch][n_q_heads] rows of 128 fp32 O, then as many fp32 lse
size_t seq_shared_workspace_bytes(int batch, int n_kv) {
  const size_t off = seq_shared_split_bytes(batch, n_kv);
  if (off == (size_t)-1) return off;
  return off + (size_t)batch * 16 * n_kv * (kHeadDim + 1) * 4;  // n_q_heads = group * n_kv, group <= 16
}

// Launch 1 streams the donor's local rows [0, prefix_len / world) once per (retrieval head, 64-row block) for the packed
// rows of all forks — the forks' rows are the "tokens" of a batch-1 no-causal partial — into fp32 (O, lse) partials.
// Launch 2 is duo_decode_fused_seq over the own slices at full_len - prefix_len; its retrieval CTAs fold those
// partials into the (O, lse) they store.
int launch_decode_fused_seq_shared(const duo_layer* L, const duo_layer* prefix, long long prefix_len,
                                   const duo_cache_state* st, const void* qkv, long long row_stride, const void* cos,
                                   const void* sin, int rope_mode, void* out, float* part_o, float* part_lse, float scale,
                                   void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  const int n_kv = d.n_full + d.n_stream;
  const size_t off = seq_shared_split_bytes(d.batch, n_kv);
  const long long rows = (long long)d.batch * n_kv * d.group;
  const size_t need = off == (size_t)-1 ? off : off + (size_t)rows * (kHeadDim + 1) * 4;
  if (need == (size_t)-1 || workspace == nullptr || workspace_bytes < need) {
    set_error("duo_decode_fused_seq_shared: workspace too small (%zu < %zu)", workspace_bytes, need);
    return DUO_EWORKSPACE;
  }
  float* pre_o = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + off);
  float* pre_lse = pre_o + rows * kHeadDim;
  duo_cache_state pst{};  // the donor's prefix rows: a plain slice, no occupancy
  pst.full_len = prefix_len / st->seq_world;
  pst.lo = d.sink;
  duo_cache_state own = *st;  // the own slices hold the positions p - prefix_len (device_state: the kernel shifts)
  own.full_len = st->full_len - prefix_len;
  return dispatch_dtype(d.dtype, [&](auto t) {
    using T = decltype(t);
    // both kernels are set up before either is enqueued: a failed call leaves nothing launched
    if (int rc = prepare_mma_kernel<T, 1, false, false, false, 4>()) return rc;
    if (int rc = prepare_mma_kernel<T, 4, true, false, false, 5>()) return rc;
    if (d.n_full > 0)
      if (int rc = launch_variant<T, 1, false, 4>(prefix, &pst, qkv, row_stride, nullptr, d.batch, scale, workspace,
                                                  workspace_bytes, stream, {pre_o, pre_lse, true}, {cos, sin, rope_mode}))
        return rc;
    return launch_variant<T, 4, true, 5>(L, &own, qkv, row_stride, out, 1, scale, workspace, workspace_bytes, stream,
                                         {part_o, part_lse, false, pre_o, pre_lse}, {cos, sin, rope_mode}, nullptr,
                                         prefix_len);
  });
}

// A chunk of forks of a sequence-sharded prompt that the wgmma kernel does not take (duo_prefill_seq_shared): the 64-row
// shard mode of duo_prefill_seq with the slice's local rows [0, prefix_rows) read from the donor, the same partition.
int launch_attn_mma_seq_shared(const duo_layer* L, const duo_layer* prefix, long long prefix_rows,
                               const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                               float* part_o, float* part_lse, int q_len, float scale, void* workspace,
                               size_t workspace_bytes, cudaStream_t stream) {
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    return launch_variant<decltype(t), 1, false, 6>(L, st, q, q_row_stride, out, q_len, scale, workspace,
                                                    workspace_bytes, stream, {part_o, part_lse}, {}, prefix,
                                                    prefix_rows);
  });
}

// Sequence-sharded chunk (duo_attention_seq: group * q_len <= 16; duo_prefill_seq: larger chunks the wgmma kernel does
// not take, on the 64-row variant): retrieval heads attend this rank's slice and report (O, lse) partials, streaming
// heads (replicated on every rank) write their final rows of `out`.
int launch_attn_mma_seq(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                        float* part_o, float* part_lse, int q_len, float scale, void* workspace, size_t workspace_bytes,
                        cudaStream_t stream) {
  const bool decode_rows = L->d.group * q_len <= 16;
  return dispatch_dtype(L->d.dtype, [&](auto t) {
    using T = decltype(t);
    return decode_rows ? launch_variant<T, 4>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes,
                                              stream, {part_o, part_lse})
                       : launch_variant<T, 1>(L, st, q, q_row_stride, out, q_len, scale, workspace, workspace_bytes,
                                              stream, {part_o, part_lse});
  });
}

}  // namespace duo
