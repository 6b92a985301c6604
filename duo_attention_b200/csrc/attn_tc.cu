// Mixed-head attention, tensor-core ("prefill") kernel for sm_90a: wgmma + TMA + mbarrier, warp-specialised.
// Replaces the FlashAttention-2 launches of duo_attn/patch/llama.py:225-267 / :364-421 for chunks of >= 128
// query tokens; both head classes run in the same launch.
//
// One CTA (1 per SM, 3 warpgroups, ~163 KB smem) processes one 128-row query tile of one q-head:
//
//   warpgroup 0      TMA producer (one thread): Q once, then K(j), V(j) tiles (128 keys x 128 dims, 128B swizzle)
//                    into 2-stage rings with separate full/empty mbarriers for K and V
//   warpgroups 1, 2  consumers, 64 query rows each, everything in registers:
//                    S = Q K^T    wgmma m64n128k16, Q and K from shared memory (K-major)
//                    mask + online softmax on the S fragment (a row lives in the 4 lanes of a quad)
//                    O += P V     wgmma m64n128k16, P from registers (the S accumulator layout IS the A fragment
//                                 layout once packed to 16 bits), V from shared memory (MN-major, transposed by wgmma)
//                    PV(j) and S(j+1) are issued back to back, so the tensor core runs one while the other drains.
//
// Masks: retrieval heads use bottom-right causal over [cache | chunk]; streaming heads attend the
// live sink/ring slots (validity table in smem) plus the staged chunk causally — see duo_b200.h.
// SEQ = true (duo_prefill_seq): the retrieval heads attend one rank's slice of a sequence-sharded cache and write
// (O, log-sum-exp) partials for the cross-rank merge; streaming heads are unchanged.
// SH = Share::DonorRows (duo_attention_shared): the retrieval keys [0, share_len) are rows of the batch-1 donor (DonorMaps),
// key j >= share_len is row j - share_len of the layer's own region; share_len is a multiple of 128, so every key tile
// lies in one region and tiles, masks and consumers are those of a row that holds all the keys itself.
// SEQ and DonorRows (duo_prefill_seq_shared, forks of a sequence-sharded prompt): the slice's local rows [0, share_len)
// are the batch-1 donor's, row j >= share_len is own row j - share_len; share_len = P / world is a multiple of 8, and the
// one tile across it is issued in 8-row pieces.  Tiles, visibility and epilogue are those of SEQ on a cache that holds
// the whole slice.
// RAGGED = true (duo_prefill_ragged): the queries are the packed chunks of the rows of a ragged batch (RaggedChunks);
// CTA (x, b) is a (kv head, q head, token tile) of row b with that row's occupancy, region and shared prefix, and the
// keys, tiles, masks, consumers and epilogue of that row's own duo_attention / duo_attention_shared launch.
#include <cstdlib>

#include "duo_common.cuh"

namespace duo {

constexpr int TC_THREADS = 384;
constexpr int TC_TILE = 128;
constexpr int TC_BOX_BYTES = TC_TILE * 128;        // 128 rows x 64 elems x 2 B = 16 KB
constexpr int TC_TILE_BYTES = 2 * TC_BOX_BYTES;    // a 128 x 128 16-bit operand tile
constexpr int TC_MAX_W = kTcMaxWindow;             // validity table size (sink + recent)
constexpr int TC_SMEM_BYTES = 5 * TC_TILE_BYTES + TC_MAX_W + 1024;  // Q K0 K1 V0 V1 + table + align

struct TcParams {
  void* out;
  long long out_batch_stride;
  int q_len, n_q_heads, group, n_full, n_stream, batch;
  int sink, recent, W;
  long long full_len, total, lo;
  float scale_log2;
  int cache_scan;
  int n_tok_tiles;  // 128-row query tiles per q-head
  // SEQ mode (duo_prefill_seq): the retrieval cache holds the block-cyclic slice of rank seq_rank (seq_local_len,
  // duo_common.cuh), full_len counts GLOBAL tokens, and retrieval heads write the fp32 normalised O and log2-domain
  // log-sum-exp of the slice to part_o [b][t][Hq][128] / part_lse [b][t][Hq] instead of `out`
  int seq_rank, seq_world, seq_block;
  float* part_o;
  float* part_lse;
};

// ---------------------------------------------------------------------------------------------
// wgmma wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Orders the compiler's reads / writes of an accumulator against the asynchronous wgmma that owns it.
__device__ __forceinline__ void wg_fence_regs(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// shared-memory matrix descriptor, SWIZZLE_128B (sm_90 GMMA descriptor layout)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= 1ull << 62;  // SWIZZLE_128B
  return d;
}

// D (+)= A[smem] * B[smem], both K-major; accum == 0 overwrites D
template <bool BF16>
__device__ __forceinline__ void wgmma_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  if constexpr (BF16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accum));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accum));
  }
}
// D += A[registers] * B[smem], B MN-major
template <bool BF16>
__device__ __forceinline__ void wgmma_rs(float (&d)[64], const uint32_t* a, uint64_t bdesc) {
  if constexpr (BF16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1));
  }
}

template <typename T>
struct TcType;
template <>
struct TcType<__nv_bfloat16> {
  static constexpr bool bf16 = true;
  __device__ static uint32_t pack(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};
template <>
struct TcType<__half> {
  static constexpr bool bf16 = false;
  __device__ static uint32_t pack(float a, float b) {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};

// barrier block in static shared memory
struct TcBarriers {
  uint64_t q_full;
  uint64_t k_full[2], k_empty[2], v_full[2], v_empty[2];
};

// (the RAGGED and donor parameters follow the others, so the parameter offsets of every instantiation are the same)
template <typename T, bool SEQ = false, Share SH = Share::None, bool RAGGED = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
duo_attn_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_fk,
                   const __grid_constant__ CUtensorMap map_fv, const __grid_constant__ CUtensorMap map_rk,
                   const __grid_constant__ CUtensorMap map_rv, const TcParams p, const __grid_constant__ RaggedChunks rc,
                   const __grid_constant__ DonorMaps dm) {
  static_assert(SH == Share::None || SH == Share::DonorRows, "the prefill kernel reads donor rows or none");
  static_assert(!(RAGGED && (SEQ || SH != Share::None)), "a ragged prefill reads sharing from row_share, and is not sharded");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ TcBarriers bars;

  uint8_t* sQ = smem;                           // 1 tile
  uint8_t* sK = smem + 1 * TC_TILE_BYTES;       // 2 stages
  uint8_t* sV = smem + 3 * TC_TILE_BYTES;       // 2 stages
  uint8_t* sValid = smem + 5 * TC_TILE_BYTES;   // [W] live-slot table (streaming heads)

  const int tid = threadIdx.x;
  const int b = blockIdx.y;

  // ---- work item ------------------------------------------------------------------------------
  // blockIdx.x enumerates (kv head, q head of the group, token tile) with retrieval heads and late tokens first
  int x = blockIdx.x;
  const int per_kvh = p.group * p.n_tok_tiles;
  const int kvh = x / per_kvh;
  x -= kvh * per_kvh;
  const int qh = kvh * p.group + x / p.n_tok_tiles;
  // RAGGED: row b's chunk, occupancy and shared prefix; its tiles are numbered as in a launch of that chunk alone, and a
  // CTA past them exits before any barrier or TMA
  int q_len = p.q_len, n_tok_tiles = p.n_tok_tiles, cache_scan = p.cache_scan, q_off = 0, donor = -1;
  long long full_len = p.full_len, total = p.total, lo = p.lo, pre_len = 0;
  if constexpr (RAGGED) {
    q_len = rc.len[b];
    n_tok_tiles = (q_len + TC_TILE - 1) / TC_TILE;
    if (x % p.n_tok_tiles >= n_tok_tiles) return;
    q_off = rc.off[b];
    full_len = rc.row_state[4 * b];
    total = rc.row_state[4 * b + 1];
    lo = rc.row_state[4 * b + 2];
    cache_scan = (int)min((long long)p.W, total);
    pre_len = ragged_chunk_share(rc, b, donor);
  }
  const int tok0 = (n_tok_tiles - 1 - (x % p.n_tok_tiles)) * TC_TILE;
  const bool is_full = kvh < p.n_full;
  const int tok_hi = min(q_len, tok0 + TC_TILE);  // exclusive
  long long a0 = 0, a1, b0 = 0, b1 = 0, base;
  if (is_full) {
    base = full_len;
    a1 = full_len + tok_hi;
    if constexpr (SEQ) a1 = seq_local_len(a1, p.seq_rank, p.seq_world, p.seq_block);  // rows of the slice
  } else {
    base = p.W;
    a1 = cache_scan;
    b0 = p.W;
    b1 = (long long)p.W + tok_hi;
  }
  const int nA = (int)((a1 - a0 + TC_TILE - 1) / TC_TILE);
  const int nB = (int)((b1 - b0 + TC_TILE - 1) / TC_TILE);
  const int n_tiles = nA + nB;  // SEQ: 0 when no row of the tile sees a key of the slice
  const CUtensorMap* mk = is_full ? &map_fk : &map_rk;
  const CUtensorMap* mv = is_full ? &map_fv : &map_rv;
  const int head_coord = is_full ? (b * p.n_full + kvh) : (b * p.n_stream + (kvh - p.n_full));
  auto tile_start = [&](int i) -> long long {
    return i < nA ? a0 + (long long)i * TC_TILE : b0 + (long long)(i - nA) * TC_TILE;
  };

  // ---- one-time setup -------------------------------------------------------------------------
  if (tid == 0) {
    prefetch_tmap(&map_q);
    prefetch_tmap(mk);
    prefetch_tmap(mv);
    if constexpr (SH == Share::DonorRows) {
      if (is_full) {
        prefetch_tmap(&dm.k);
        prefetch_tmap(&dm.v);
      }
    }
    mbar_init(&bars.q_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bars.k_full[s], 1);
      mbar_init(&bars.k_empty[s], 256);  // every consumer thread releases the stage after its wgmma completed
      mbar_init(&bars.v_full[s], 1);
      mbar_init(&bars.v_empty[s], 256);
    }
    fence_barrier_init();
  }
  if (!is_full) {
    for (int j = tid; j < p.W; j += TC_THREADS) sValid[j] = stream_slot_valid(j, p.sink, p.recent, total, lo) ? 1 : 0;
  }
  __syncthreads();

  if (tid < 128) {
    // ======================= TMA producer =======================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if constexpr (SEQ) {
      if (n_tiles == 0) return;  // no Q, no K/V: the consumers write the empty rows without waiting
    }
    if (tid == 0) {
      mbar_expect_tx(&bars.q_full, TC_TILE_BYTES);
      const int q_row = RAGGED ? q_off + tok0 : tok0, q_b = RAGGED ? 0 : b;  // RAGGED: map_q spans the packed tokens
      tma_load_3d(sQ, &map_q, &bars.q_full, qh * kHeadDim, q_row, q_b);
      tma_load_3d(sQ + TC_BOX_BYTES, &map_q, &bars.q_full, qh * kHeadDim + 64, q_row, q_b);
      // retrieval tiles that can come from two regions (DonorRows; RAGGED: a sharer's prefix in the donor's region of
      // the pool, its own keys in its region, both through the pool map at head 0) go through tma_key_operand, the
      // plain instantiations load the own rows directly
      constexpr bool kRegions = SH == Share::DonorRows || RAGGED;
      KeyRegions kr{0, 0, 0, 0, head_coord};
      if constexpr (SH == Share::DonorRows) {
        if (is_full) kr = {dm.rows, 0, 0, kvh, head_coord};
      }
      if constexpr (RAGGED) {
        if (is_full && rc.row_geom)
          kr = {pre_len, pre_len > 0 ? ragged_pool_row(rc, donor, p.n_full, kvh, 0) : 0,
                ragged_pool_row(rc, b, p.n_full, kvh, 0), 0, 0};
      }
      const CUtensorMap* dk = SH == Share::DonorRows ? &dm.k : mk;
      const CUtensorMap* dv = SH == Share::DonorRows ? &dm.v : mv;
      auto load = [&](uint8_t* dst, const CUtensorMap* own, const CUtensorMap* donor, const CUtensorMap* donor8,
                      const CUtensorMap* own8, uint64_t* bar, int t0) {
        if constexpr (kRegions) {
          tma_key_operand<TC_TILE, SEQ>(dst, TC_BOX_BYTES, donor, own, donor8, own8, bar, t0, kr);
        } else {
          tma_load_3d(dst, own, bar, 0, t0, head_coord);
          tma_load_3d(dst + TC_BOX_BYTES, own, bar, 64, t0, head_coord);
        }
      };
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        const int t0 = (int)tile_start(j);  // (a TMA row coordinate)
        mbar_wait(&bars.k_empty[st], ph ^ 1);
        mbar_expect_tx(&bars.k_full[st], TC_TILE_BYTES);
        load(sK + st * TC_TILE_BYTES, mk, dk, &dm.k8, &dm.own_k8, &bars.k_full[st], t0);
        mbar_wait(&bars.v_empty[st], ph ^ 1);
        mbar_expect_tx(&bars.v_full[st], TC_TILE_BYTES);
        load(sV + st * TC_TILE_BYTES, mv, dv, &dm.v8, &dm.own_v8, &bars.v_full[st], t0);
      }
    }
    return;
  }

  // ======================= consumer warpgroups =======================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
  constexpr bool kBf16 = TcType<T>::bf16;
  const int wg = (tid >> 7) - 1;              // 0, 1: query rows [64 wg, 64 wg + 64) of the tile
  const int wt = tid & 127;
  const int quad = wt & 3;                    // column pair inside each 8-column block
  const int row0 = wg * 64 + (wt >> 5) * 16 + ((wt & 31) >> 2);  // this thread's rows: row0, row0 + 8
  const float c = p.scale_log2;
  long long min_limit = base + tok0 + wg * 64;  // last visible key of this warpgroup's first row
  int tok[2];
  bool row_ok[2];
  long long limit[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    tok[i] = tok0 + row0 + 8 * i;
    row_ok[i] = tok[i] < q_len;
    limit[i] = base + tok[i];
  }
  // SEQ retrieval heads: row t sees the local rows of positions <= full_len + t; the slice is in position order, so that
  // is a prefix of the slice too (-1: the row sees no key of it)
  auto seq_last_key = [&](int t) { return seq_local_len(p.full_len + t + 1, p.seq_rank, p.seq_world, p.seq_block) - 1; };
  if constexpr (SEQ) {
    if (is_full) {
      min_limit = seq_last_key(tok0 + wg * 64);
#pragma unroll
      for (int i = 0; i < 2; ++i) limit[i] = seq_last_key(tok[i]);
    }
  }

  const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128, k_addr = smem_u32(sK), v_addr = smem_u32(sV);
  auto issue_s = [&](float (&s)[64], int st) {
    const uint32_t ka = k_addr + st * TC_TILE_BYTES;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t off = (kk >> 2) * TC_BOX_BYTES + (kk & 3) * 32;
      wgmma_ss<kBf16>(s, make_smem_desc(q_addr + off, 16, 1024), make_smem_desc(ka + off, 16, 1024), kk > 0);
    }
  };
  auto issue_pv = [&](float (&o)[64], const uint32_t (&pk)[32], int st) {
    const uint32_t va = v_addr + st * TC_TILE_BYTES;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_rs<kBf16>(o, &pk[4 * kk], make_smem_desc(va + kk * 2048, TC_BOX_BYTES, 1024));
  };

  float s[64], o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};  // this thread's share of the row sums (its 32 columns of every tile)

  // SEQ retrieval heads: fp32 normalised O and m * scale * log2(e) + log2(l) of the slice (lse = -inf, O = 0 for a row
  // that sees no key of it); rows past q_len are not stored
  auto store_partial = [&](int i, float inv, float l) {
    if (!row_ok[i]) return;
    const long long row = ((long long)b * p.q_len + tok[i]) * p.n_q_heads + qh;
#pragma unroll
    for (int nb = 0; nb < 16; ++nb)
      *reinterpret_cast<float2*>(p.part_o + row * kHeadDim + nb * 8 + quad * 2) =
          make_float2(o[nb * 4 + 2 * i] * inv, o[nb * 4 + 2 * i + 1] * inv);
    if (quad == 0) p.part_lse[row] = l > 0.f ? m_run[i] * c + log2f(l) : -INFINITY;
  };
  if constexpr (SEQ) {
    if (n_tiles == 0) {
      store_partial(0, 0.f, 0.f);
      store_partial(1, 0.f, 0.f);
      return;
    }
  }
  mbar_wait(&bars.q_full, 0);
  mbar_wait(&bars.k_full[0], 0);
  wg_fence();
  issue_s(s, 0);
  wg_commit();
  wg_wait<0>();
  wg_fence_regs(s);
  mbar_arrive(&bars.k_empty[0]);

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    const long long j0 = tile_start(j);
    const long long jend = (j < nA) ? a1 : b1;
    const bool cache_seg = (!is_full) && (j < nA);
    const bool need_mask = cache_seg || (j0 + TC_TILE > jend) || (j0 + TC_TILE - 1 > min_limit);
    if (need_mask) {
#pragma unroll
      for (int nb = 0; nb < 16; ++nb) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const long long jj = j0 + nb * 8 + quad * 2 + e;
          bool slot_ok = jj < jend;
          if (cache_seg) slot_ok = slot_ok && (jj < p.W) && (sValid[jj < p.W ? jj : 0] != 0);
#pragma unroll
          for (int i = 0; i < 2; ++i)
            if (!(slot_ok && row_ok[i] && jj <= limit[i])) s[nb * 4 + 2 * i + e] = -INFINITY;
        }
      }
    }
    // ---- online softmax on the fragment: row i of this thread = s[nb*4 + 2i + {0,1}], nb = 0..15
    uint32_t pk[32];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < 16; ++nb) mx = fmaxf(mx, fmaxf(s[nb * 4 + 2 * i], s[nb * 4 + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[i], mx);
      const float alpha = (m_new == -INFINITY) ? 1.f : fast_exp2((m_run[i] - m_new) * c);
      const float mref_c = (m_new == -INFINITY) ? 0.f : m_new * c;
      m_run[i] = m_new;
      float rs = 0.f;
#pragma unroll
      for (int nb = 0; nb < 16; ++nb) {
        const float p0 = fast_exp2(__fmaf_rn(s[nb * 4 + 2 * i], c, -mref_c));
        const float p1 = fast_exp2(__fmaf_rn(s[nb * 4 + 2 * i + 1], c, -mref_c));
        rs += p0 + p1;  // l accumulates the unrounded p in fp32, like FA2
        pk[nb * 2 + i] = TcType<T>::pack(p0, p1);
        o[nb * 4 + 2 * i] *= alpha;
        o[nb * 4 + 2 * i + 1] *= alpha;
      }
      l_run[i] = l_run[i] * alpha + rs;
    }
    // ---- O += P V(j), then S = Q K(j+1)^T behind it on the tensor core
    mbar_wait_spin(&bars.v_full[st], ph);
    wg_fence();
    issue_pv(o, pk, st);
    wg_commit();
    const bool more = j + 1 < n_tiles;
    if (more) {
      const int st1 = (j + 1) & 1;
      mbar_wait_spin(&bars.k_full[st1], ((j + 1) >> 1) & 1);
      wg_fence();  // the softmax rewrote the S registers since the fence before PV(j)
      issue_s(s, st1);
      wg_commit();
    }
    wg_wait<0>();
    wg_fence_regs(o);
    wg_fence_regs(s);
    mbar_arrive(&bars.v_empty[st]);
    if (more) mbar_arrive(&bars.k_empty[(j + 1) & 1]);
  }

  // ---- epilogue: O / l -> global ----------------------------------------------------------------
  if constexpr (SEQ) {
    if (is_full) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float l = l_run[i];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        store_partial(i, l > 0.f ? 1.f / l : 0.f, l);
      }
      return;
    }
  }
  // RAGGED: `out` holds the packed tokens, row b's from q_off
  T* out_b = reinterpret_cast<T*>(p.out) + (RAGGED ? (long long)q_off * p.n_q_heads * kHeadDim : (long long)b * p.out_batch_stride);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = l > 0.f ? 1.f / l : 0.f;
    if (row_ok[i]) {
      T* dst = out_b + ((long long)tok[i] * p.n_q_heads + qh) * kHeadDim + quad * 2;
#pragma unroll
      for (int nb = 0; nb < 16; ++nb)
        *reinterpret_cast<uint32_t*>(dst + nb * 8) = TcType<T>::pack(o[nb * 4 + 2 * i] * inv, o[nb * 4 + 2 * i + 1] * inv);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();  // api.cu

bool tc_prefill_supported(const duo_layer* L, const duo_cache_state* st, int q_len) {
  (void)st;
  if (L->d.kv_format != DUO_KV_SAME) return false;
  if (q_len < TC_TILE) return false;
  if (L->d.sink + L->d.recent > TC_MAX_W) return false;
  return true;
}

// Q inside the fused qkv buffer, [batch][rows][row width] with 128-row boxes; rows past `rows` read as zero
static int encode_q_map(CUtensorMap* map_q, const duo_layer_desc& d, const void* q, long long row_stride,
                        long long rows, long long batch) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return DUO_ECUDA;
  cuuint64_t dims[3] = {(cuuint64_t)row_stride, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[2] = {(cuuint64_t)row_stride * 2, (cuuint64_t)row_stride * 2 * (cuuint64_t)rows};
  cuuint32_t box[3] = {64, TC_TILE, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map_q, d.dtype == DUO_DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                  const_cast<void*>(q), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(q) failed with CUresult %d", (int)r);
    return DUO_ECUDA;
  }
  return DUO_OK;
}

// The fields of TcParams every launch fills: `out` and the layer's head geometry (as fill_common_params does for the
// bandwidth kernels)
static TcParams tc_common_params(const duo_layer_desc& d, void* out, float scale) {
  TcParams p{};
  p.out = out;
  p.n_q_heads = (d.n_full + d.n_stream) * d.group;
  p.group = d.group;
  p.n_full = d.n_full;
  p.n_stream = d.n_stream;
  p.batch = d.batch;
  p.sink = d.sink;
  p.recent = d.recent;
  p.W = d.sink + d.recent;
  p.scale_log2 = scale * 1.4426950408889634f;
  return p;
}

// SEQ: the retrieval heads attend the rank's slice described by st and report (part_o, part_lse); see TcParams.
// DonorRows: the first share_len retrieval keys (SEQ: local rows of the slice) are rows of `prefix` (see
// duo_attn_tc_kernel).
template <bool SEQ, Share SH = Share::None>
static int launch_tc(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                     float* part_o, float* part_lse, int q_len, float scale, cudaStream_t stream,
                     const duo_layer* prefix = nullptr, long long share_len = 0) {
  const duo_layer_desc& d = L->d;
  CUtensorMap map_q;
  if (int rc = encode_q_map(&map_q, d, q, q_row_stride, q_len, d.batch)) return rc;
  TcParams p = tc_common_params(d, out, scale);
  p.out_batch_stride = (long long)q_len * p.n_q_heads * kHeadDim;
  p.q_len = q_len;
  p.full_len = st->full_len;
  p.total = st->total;
  p.lo = st->lo;
  p.cache_scan = (int)std::min<long long>(p.W, st->total);
  p.n_tok_tiles = (q_len + TC_TILE - 1) / TC_TILE;
  p.seq_rank = st->seq_rank;
  p.seq_world = st->seq_world;
  p.seq_block = st->seq_block;
  p.part_o = part_o;
  p.part_lse = part_lse;
  const dim3 grid(p.n_q_heads * p.n_tok_tiles, d.batch);
  const KvMaps m = kv_maps(L, true);
  DonorMaps dm;
  if (int rc = donor_maps(L, prefix, share_len, true, dm)) return rc;
  return dispatch_dtype(d.dtype, [&](auto t) {
    auto kern = duo_attn_tc_kernel<decltype(t), SEQ, SH>;
    static unsigned long long attr_mask = 0;  // per kernel instantiation, one bit per device
    if (int rc = ensure_dyn_smem(kern, TC_SMEM_BYTES, &attr_mask)) return rc;
    kern<<<grid, TC_THREADS, TC_SMEM_BYTES, stream>>>(map_q, *m.fk, *m.fv, *m.rk, *m.rv, p, RaggedChunks{}, dm);
    DUO_CUDA_TRY(cudaGetLastError());
    return DUO_OK;
  });
}

int launch_rope_append_ragged(const duo_layer* L, const RaggedChunks& rc, void* qkv, long long row_stride,
                              const void* cos, const void* sin, int rope_mode, cudaStream_t stream);  // kv_ops.cu
int launch_stream_commit_ragged(const duo_layer* L, const RaggedChunks& rc, cudaStream_t stream);     // kv_ops.cu

// Batched ragged prefill (duo_prefill_ragged, arguments checked there): RoPE + append of every row's chunk, the wgmma
// attention of all rows in one launch, the ring commit.  Everything that can fail is set up before the first launch.
int launch_prefill_ragged(const duo_layer* L, const RaggedChunks& rc, void* qkv, long long row_stride, const void* cos,
                          const void* sin, int rope_mode, void* out, float scale, cudaStream_t stream) {
  const duo_layer_desc& d = L->d;
  const int n_tok = rc.off[rc.batch];
  int max_tiles = 0;
  for (int b = 0; b < rc.batch; ++b) max_tiles = std::max(max_tiles, (rc.len[b] + TC_TILE - 1) / TC_TILE);
  if (n_tok == 0) return DUO_OK;
  CUtensorMap map_q;  // the packed tokens: {row width, T, 1}
  if (int rc2 = encode_q_map(&map_q, d, qkv, row_stride, n_tok, 1)) return rc2;
  TcParams p = tc_common_params(d, out, scale);
  p.n_tok_tiles = max_tiles;  // the grid's tiles per q-head; row b's CTAs past its own tiles exit
  const dim3 grid(p.n_q_heads * max_tiles, d.batch);
  const KvMaps m = kv_maps(L, true);
  return dispatch_dtype(d.dtype, [&](auto t) {
    auto kern = duo_attn_tc_kernel<decltype(t), false, Share::None, true>;
    static unsigned long long attr_mask = 0;
    if (int rc2 = ensure_dyn_smem(kern, TC_SMEM_BYTES, &attr_mask)) return rc2;
    if (int rc2 = launch_rope_append_ragged(L, rc, qkv, row_stride, cos, sin, rope_mode, stream)) return rc2;
    kern<<<grid, TC_THREADS, TC_SMEM_BYTES, stream>>>(map_q, *m.fk, *m.fv, *m.rk, *m.rv, p, rc, DonorMaps{});
    DUO_CUDA_TRY(cudaGetLastError());
    return launch_stream_commit_ragged(L, rc, stream);
  });
}

int launch_attn_tc(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                   int q_len, float scale, cudaStream_t stream) {
  return launch_tc<false>(L, st, q, q_row_stride, out, nullptr, nullptr, q_len, scale, stream);
}

// Sequence-sharded prefill chunk (duo_prefill_seq): retrieval heads report slice partials, streaming heads write `out`.
int launch_attn_tc_seq(const duo_layer* L, const duo_cache_state* st, const void* q, long long q_row_stride, void* out,
                       float* part_o, float* part_lse, int q_len, float scale, cudaStream_t stream) {
  return launch_tc<true>(L, st, q, q_row_stride, out, part_o, part_lse, q_len, scale, stream);
}

// A chunk of a row whose first share_len retrieval keys are rows of `prefix` (duo_attention_shared).
int launch_attn_tc_shared(const duo_layer* L, const duo_layer* prefix, long long share_len, const duo_cache_state* st,
                          const void* q, long long q_row_stride, void* out, int q_len, float scale, cudaStream_t stream) {
  return launch_tc<false, Share::DonorRows>(L, st, q, q_row_stride, out, nullptr, nullptr, q_len, scale, stream, prefix,
                                           share_len);
}

// A chunk of forks of a sequence-sharded prompt (duo_prefill_seq_shared): the slice's local rows [0, prefix_rows) are
// the donor's, the rest the forks' own slices; retrieval heads report slice partials, streaming heads write `out`.
int launch_attn_tc_seq_shared(const duo_layer* L, const duo_layer* prefix, long long prefix_rows,
                              const duo_cache_state* st, const void* q, long long q_row_stride, void* out, float* part_o,
                              float* part_lse, int q_len, float scale, cudaStream_t stream) {
  return launch_tc<true, Share::DonorRows>(L, st, q, q_row_stride, out, part_o, part_lse, q_len, scale, stream, prefix,
                                          prefix_rows);
}

}  // namespace duo
