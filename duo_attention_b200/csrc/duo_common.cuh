// Shared device helpers (sm_90a): mbarrier, TMA, ldmatrix, mma.sync wrappers + host-side
// error plumbing.  Everything here is hand-written PTX; no CUTLASS/CuTe.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/duo_b200.h"

namespace duo {

constexpr int kHeadDim = 128;
constexpr int kTcMaxWindow = 2048;  // the most sink + recent slots the wgmma prefill kernel's validity table holds

// ---------------------------------------------------------------------------------------------
// host-side error handling
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
#define DUO_CUDA_TRY(expr)                                   \
  do {                                                       \
    cudaError_t _e = (expr);                                 \
    if (_e != cudaSuccess) return ::duo::cuda_fail(_e, #expr); \
  } while (0)

// ---------------------------------------------------------------------------------------------
// the opaque per-layer handle
// ---------------------------------------------------------------------------------------------
struct LayerMaps {
  // 3-D maps {head_dim, slots, batch*heads}; box {64 elems, tile rows, 1}; SWIZZLE_128B
  CUtensorMap full_k64, full_v64;    // 64-row boxes (mma.sync bandwidth kernel)
  CUtensorMap ring_k64, ring_v64;
  CUtensorMap full_k128, full_v128;  // 128-row boxes (wgmma prefill kernel)
  CUtensorMap ring_k128, ring_v128;
};

}  // namespace duo

struct duo_layer {
  duo_layer_desc d;
  duo::LayerMaps maps;
  bool has_full_maps;
  bool has_ring_maps;
  int64_t pool_tokens;  // > 0: a pooled ragged layer (duo_layer_create_pooled), full maps span the pool
};

namespace duo {

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a lost TMA transaction / missing arrival must not hang the GPU.  After 2^26 failed polls (a failed
// try_wait suspends the thread for an implementation-defined interval first, so this is seconds to a minute) the
// kernel traps, which surfaces as a CUDA launch failure (DUO_ECUDA at the next API call) instead of a wedged device.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++polls == (1u << 26)) asm volatile("trap;");
  }
}
// Unbounded spin for register-starved consumers whose producer side is already bounded (a trap anywhere ends the grid).
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// TMA tiled 3-D load global -> shared, completion on an mbarrier (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// One ROWS-key operand (K or V, both 64-column halves, box_bytes apart) of a retrieval tile of a fork of a
// sequence-sharded prompt (duo_prefill_seq_shared), starting at local row t0 of the logical slice: rows j < c are the
// donor's (a batch-1 handle: head coordinate kvh), rows j >= c are own rows j - c (head coordinate hc).  c is a multiple
// of 8 but not of ROWS, so a tile across it is issued in 8-row pieces (pre8 / own8: 8-row boxes), each from its source.
// An 8-row x 128-byte piece is one SWIZZLE_128B atom: pieces at 1024-byte steps land as the whole box would, and the
// bytes the tile delivers are the same.
template <int ROWS>
__device__ __forceinline__ void tma_fork_operand(uint8_t* dst, int box_bytes, const CUtensorMap* pre,
                                                 const CUtensorMap* own, const CUtensorMap* pre8, const CUtensorMap* own8,
                                                 uint64_t* bar, long long t0, long long c, int kvh, int hc) {
  if (t0 + ROWS <= c || t0 >= c) {
    const bool p = t0 < c;
    const CUtensorMap* m = p ? pre : own;
    const int r0 = (int)(p ? t0 : t0 - c), h = p ? kvh : hc;
    tma_load_3d(dst, m, bar, 0, r0, h);
    tma_load_3d(dst + box_bytes, m, bar, 64, r0, h);
    return;
  }
  for (int k = 0; k < ROWS / 8; ++k) {
    const long long r = t0 + 8 * k;
    const bool p = r < c;
    const CUtensorMap* m = p ? pre8 : own8;
    const int r0 = (int)(p ? r : r - c), h = p ? kvh : hc;
    tma_load_3d(dst + k * 1024, m, bar, 0, r0, h);
    tma_load_3d(dst + box_bytes + k * 1024, m, bar, 64, r0, h);
  }
}
__device__ __forceinline__ void tma_load_3d_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                                 int c2, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, "
      "%4, %5}], [%2], %6;" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

__device__ __forceinline__ void ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}

template <typename T>
struct MmaOp;
template <>
struct MmaOp<__nv_bfloat16> {
  __device__ __forceinline__ static void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  __device__ __forceinline__ static uint32_t pack(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};
template <>
struct MmaOp<__half> {
  __device__ __forceinline__ static void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  __device__ __forceinline__ static uint32_t pack(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};

// ---------------------------------------------------------------------------------------------
// RoPE element arithmetic, shared by rope_append_kernel (kv_ops.cu) and the fused decode kernel (attn_mma.cu) so that
// both produce the same bits.  `rot` is the rotate_half partner with its sign (exact in T).
//   HF  : T(T(x*cos) + T(rot*sin))   — transformers' apply_rotary_pos_emb on T tensors (llama.py:177-184)
//   fp32: T(x*cos + rot*sin), fp32 tables, one rounding (flashinfer semantics, flashinfer_utils.py:29-59)
// ---------------------------------------------------------------------------------------------
template <typename T>
struct RopeCvt;
template <>
struct RopeCvt<__nv_bfloat16> {
  __device__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <>
struct RopeCvt<__half> {
  __device__ static float to_f(__half v) { return __half2float(v); }
  __device__ static __half from_f(float v) { return __float2half_rn(v); }
};
template <typename T>
__device__ __forceinline__ float rope_hf(float x, float rot, float c, float s) {
  const float a = RopeCvt<T>::to_f(RopeCvt<T>::from_f(__fmul_rn(x, c)));
  const float r = RopeCvt<T>::to_f(RopeCvt<T>::from_f(__fmul_rn(rot, s)));
  return __fadd_rn(a, r);  // the caller's conversion to T is the third rounding
}
__device__ __forceinline__ float rope_f32(float x, float rot, float c, float s) {
  return __fmaf_rn(rot, s, __fmul_rn(x, c));
}

// RoPE of 8 consecutive head_dim elements d .. d+7 (d < 64) and their partners d+64 .. d+71, arithmetic of
// rope_append_kernel (kv_ops.cu): HF mode rounds every product and the sum to T, fp32 mode rounds once.
template <typename T>
__device__ __forceinline__ void rope8(uint4& lo, uint4& hi, const void* cos, const void* sin, int mode, int tok, int d) {
  T* xl = reinterpret_cast<T*>(&lo);
  T* xh = reinterpret_cast<T*>(&hi);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
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

// ---------------------------------------------------------------------------------------------
// One 128-element row held 4-per-lane by a warp (lane l: elements 4l .. 4l+3): RoPE and INT4 K1 quantisation.
// Shared by rope_append_kernel (kv_ops.cu) and the fused INT4 decode kernel (attn_int4.cu): same bits from both.
// ---------------------------------------------------------------------------------------------
template <typename T>
struct alignas(8) Vec4 {
  T v[4];
};

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// RoPE of token `t` (row t of the cos / sin tables of this chunk) on a warp-held row; every lane must call.
template <typename T>
__device__ __forceinline__ void rope_row4(Vec4<T>& xv, int lane, int t, const void* cos, const void* sin, int mode) {
  // rotate_half partner: element i pairs with i +- 64  <=> lane +- 16
  Vec4<T> pv;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float mine = RopeCvt<T>::to_f(xv.v[i]);
    const float other = __shfl_xor_sync(0xffffffffu, mine, 16);
    pv.v[i] = RopeCvt<T>::from_f(lane < 16 ? -other : other);
  }
  if (mode == DUO_ROPE_HF) {
    const Vec4<T> cv = *reinterpret_cast<const Vec4<T>*>(reinterpret_cast<const T*>(cos) + (long long)t * kHeadDim + lane * 4);
    const Vec4<T> sv = *reinterpret_cast<const Vec4<T>*>(reinterpret_cast<const T*>(sin) + (long long)t * kHeadDim + lane * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      xv.v[i] = RopeCvt<T>::from_f(rope_hf<T>(RopeCvt<T>::to_f(xv.v[i]), RopeCvt<T>::to_f(pv.v[i]), RopeCvt<T>::to_f(cv.v[i]),
                                              RopeCvt<T>::to_f(sv.v[i])));
  } else {
    const float4 cv = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(cos) + (long long)t * kHeadDim + lane * 4);
    const float4 sv = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(sin) + (long long)t * kHeadDim + lane * 4);
    const float c[4] = {cv.x, cv.y, cv.z, cv.w};
    const float s[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
      xv.v[i] = RopeCvt<T>::from_f(rope_f32(RopeCvt<T>::to_f(xv.v[i]), RopeCvt<T>::to_f(pv.v[i]), c[i], s[i]));
  }
}

// K1 arithmetic (demo/quantize_int4.cu:73-144) for one 128-element group held 4-per-lane (fp16-representable values
// in x[]).  Writes 2 packed bytes per lane; lane 0 writes scale / zero.
__device__ __forceinline__ void quant_row_int4(const float (&x)[4], int lane, uint8_t* packed_row, __half* scale_p,
                                               __half* zero_p) {
  float mn = fminf(fminf(x[0], x[1]), fminf(x[2], x[3]));
  float mx = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3]));
  mn = warp_min(mn);
  mx = warp_max(mx);
  const float scale = __fadd_rn(__fdiv_rn(__fsub_rn(mx, mn), 15.0f), 1e-8f);
  const float zero = mn;
  uint32_t q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float qf = __fdiv_rn(__fsub_rn(x[i], zero), scale);
    qf = roundf(qf);
    qf = fminf(fmaxf(qf, 0.0f), 15.0f);
    q[i] = (uint32_t)qf;
  }
  const uint16_t two = (uint16_t)(((q[0] << 4) | q[1]) | (((q[2] << 4) | q[3]) << 8));
  *reinterpret_cast<uint16_t*>(packed_row + 2 * lane) = two;
  if (lane == 0) {
    *scale_p = __float2half_rn(scale);
    *zero_p = __float2half_rn(zero);
  }
}

// fp32 pair helpers: two independent round-to-nearest ops (sm_90 has no packed fp32 instructions)
__device__ __forceinline__ void fma2(float& o0, float& o1, float a0, float a1, float b0, float b1, float c0, float c1) {
  o0 = __fmaf_rn(a0, b0, c0);
  o1 = __fmaf_rn(a1, b1, c1);
}
__device__ __forceinline__ void add2(float& o0, float& o1, float a0, float a1, float b0, float b1) {
  o0 = __fadd_rn(a0, b0);
  o1 = __fadd_rn(a1, b1);
}
__device__ __forceinline__ void mul2(float& o0, float& o1, float a0, float a1, float b0, float b1) {
  o0 = __fmul_rn(a0, b0);
  o1 = __fmul_rn(a1, b1);
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Is ring/sink slot `j` (< sink+recent) of a streaming head holding a live token?
// See duo_cache_state in duo_b200.h.
__device__ __forceinline__ bool stream_slot_valid(int j, int sink, int recent, long long total, long long lo) {
  if (j < sink) return j < total;
  if (total <= sink) return false;
  long long last = total - 1;
  long long r = j - sink;
  long long diff = (last - sink - r) % recent;
  if (diff < 0) diff += recent;
  long long p = last - diff;
  return p >= lo;
}

// Split-KV merge: one warp merges its share of the `splits` partials (splits warp, warp+4, ...) for up to FOUR rows
// at once, i.e. 16 independent 512-byte loads in flight per iteration.  (A row-at-a-time loop costs splits/16
// dependent L2 round trips PER ROW, which dominated decode launches with a single retrieval head.)
//   po  : [splits][ROWS][128] un-normalised partial outputs, pml : [splits][ROWS][2] (max in log2 domain, sum)
//   rows r0 .. r0+nr-1 (nr <= 4); results: acc[q] (this lane's 4 output dims), mm[q], ll[q]
template <int ROWS>
__device__ __forceinline__ void split_merge_rows4(const float* po, const float* pml, int splits, int warp, int lane,
                                                  int r0, int nr, float4 (&acc)[4], float (&mm)[4], float (&ll)[4]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    mm[q] = -INFINITY;
    ll[q] = 0.f;
  }
  for (int s0 = warp; s0 < splits; s0 += 16) {
    float ms[4][4], ls[4][4];
    float4 vs[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int s2 = s0 + 4 * u;
      const bool sok = s2 < splits;
      const int sc2 = sok ? s2 : s0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const bool ok = sok && q < nr;
        const int r = r0 + (q < nr ? q : 0);
        ms[u][q] = ok ? __ldcg(&pml[(sc2 * ROWS + r) * 2]) : -INFINITY;
        ls[u][q] = __ldcg(&pml[(sc2 * ROWS + r) * 2 + 1]);
        vs[u][q] = __ldcg(reinterpret_cast<const float4*>(&po[((long long)sc2 * ROWS + r) * 128 + lane * 4]));
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (ms[u][q] == -INFINITY) continue;
        const float mn = fmaxf(mm[q], ms[u][q]);
        const float fo = (mm[q] == -INFINITY) ? 0.f : fast_exp2(mm[q] - mn);
        const float fn = fast_exp2(ms[u][q] - mn);
        acc[q].x = acc[q].x * fo + vs[u][q].x * fn;
        acc[q].y = acc[q].y * fo + vs[u][q].y * fn;
        acc[q].z = acc[q].z * fo + vs[u][q].z * fn;
        acc[q].w = acc[q].w * fo + vs[u][q].w * fn;
        ll[q] = ll[q] * fo + ls[u][q] * fn;
        mm[q] = mn;
      }
    }
  }
}


// ---------------------------------------------------------------------------------------------
// Split-KV publish / merge protocol shared by the three bandwidth kernels (attn_mma.cu, attn_int4.cu x2).
//
// Every CTA of a (batch, kv head, row block) "item" writes its partial (un-normalised O, running max in the log2
// domain, row sum) to the workspace.  Merging is HIERARCHICAL: the splits of an item form groups of kMergeGroup; the
// last CTA of a group to arrive merges that group into a level-2 partial, the last GROUP to finish merges the level-2
// partials into the result.  Group merges happen while other CTAs are still streaming keys, so only the final merge
// of <= splits/16 partials is on the critical path.
// ---------------------------------------------------------------------------------------------
constexpr int kMergeGroup = 16;

struct SplitWs {        // device pointers into the caller's workspace
  int* counters;        // [items][1 + n_groups]  (top-level arrival count, then one per group); zero between launches
  float* ws_ml;         // [items][splits][ROWS][2]
  float* ws_o;          // [items][splits][ROWS][128]
  float* g_ml;          // [items][n_groups][ROWS][2]     level-2 partials
  float* g_o;           // [items][n_groups][ROWS][128]
  int n_groups;
};

inline int split_groups(int splits) { return splits <= kMergeGroup ? 1 : (splits + kMergeGroup - 1) / kMergeGroup; }

// The arrival counters live in a FIXED region at the start of the workspace (they must stay zero between launches, and
// launches of different geometry — layers with different numbers of retrieval heads, decode steps and chunks — share
// one workspace: a geometry-dependent counter region would overlap partial data written by an earlier launch).
constexpr size_t kSplitCounterBytes = 64 * 1024;

// What a launch keeps in the workspace: after the counter region, `parts` level-1 partials ([rows][2] then [rows][128]
// floats, each array 256-byte aligned) and `groups` level-2 partials of the same shape.
struct SplitWsLayout {
  long long items;   // retrieval items; each owns 1 + n_groups arrival counters
  int n_groups;      // per-item stride of the counters and the level-2 partials
  long long parts;   // level-1 partials
  long long groups;  // level-2 partials (0: the splits of an item are merged in one level)
  int rows;          // rows per partial
};

// layout of a launch whose `items` items take `splits` splits each
inline SplitWsLayout split_ws_layout(long long items, int splits, int rows) {
  const int ng = split_groups(splits);
  return {items, ng, items * splits, ng > 1 ? items * ng : 0, rows};
}

inline size_t split_ws_region(long long partials, int floats_per_partial) {
  return ((size_t)partials * floats_per_partial * 4 + 255) / 256 * 256;
}

// bytes of workspace the layout needs; SIZE_MAX if it has too many counters
inline size_t split_ws_bytes(const SplitWsLayout& l) {
  if ((size_t)l.items * (1 + l.n_groups) * 4 > kSplitCounterBytes) return (size_t)-1;
  return kSplitCounterBytes + split_ws_region(l.parts, l.rows * 2) + split_ws_region(l.parts, l.rows * 128) +
         split_ws_region(l.groups, l.rows * 2) + split_ws_region(l.groups, l.rows * 128) + 256;
}

// Points `w` into `workspace` by the layout; DUO_EWORKSPACE (reported as `who`) if the workspace is too small.
inline int split_ws_carve(SplitWs& w, const SplitWsLayout& l, void* workspace, size_t workspace_bytes, const char* who) {
  const size_t need = split_ws_bytes(l);
  if (need == (size_t)-1 || workspace == nullptr || workspace_bytes < need) {
    set_error("%s: workspace too small (%zu < %zu)", who, workspace_bytes, need);
    return DUO_EWORKSPACE;
  }
  uint8_t* p = reinterpret_cast<uint8_t*>(workspace);
  w.n_groups = l.n_groups;
  w.counters = reinterpret_cast<int*>(p);
  p += kSplitCounterBytes;
  w.ws_ml = reinterpret_cast<float*>(p);
  p += split_ws_region(l.parts, l.rows * 2);
  w.ws_o = reinterpret_cast<float*>(p);
  p += split_ws_region(l.parts, l.rows * 128);
  if (l.groups > 0) {
    w.g_ml = reinterpret_cast<float*>(p);
    p += split_ws_region(l.groups, l.rows * 2);
    w.g_o = reinterpret_cast<float*>(p);
  }
  return DUO_OK;
}

// CTA-wide (128 threads) merge of `n` partials po [n][ROWS][128] / pml [n][ROWS][2] for rows [0, rows):
// emit(r, d, a0, a1, mm, ll) receives the UN-NORMALISED sums of dims d, d+1 and the merged (max, row sum).
// cm_o: [4][16][128] floats, cm_ml: [4][16][2] floats of shared memory.
template <int ROWS, typename Emit>
__device__ __forceinline__ void merge_partials_cta(const float* po, const float* pml, int n, int rows, float* cm_o,
                                                   float* cm_ml, Emit emit) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int rg = 0; rg < rows; rg += 16) {
    const int rg_n = min(16, rows - rg);
    for (int rr0 = 0; rr0 < rg_n; rr0 += 4) {
      const int nr = min(4, rg_n - rr0);
      float4 acc4[4];
      float mm4[4], ll4[4];
      split_merge_rows4<ROWS>(po, pml, n, warp, lane, rg + rr0, nr, acc4, mm4, ll4);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q < nr) {
          *reinterpret_cast<float4*>(&cm_o[(warp * 16 + rr0 + q) * 128 + lane * 4]) = acc4[q];
          if (lane == 0) {
            cm_ml[(warp * 16 + rr0 + q) * 2] = mm4[q];
            cm_ml[(warp * 16 + rr0 + q) * 2 + 1] = ll4[q];
          }
        }
      }
    }
    __syncthreads();
    for (int idx = tid; idx < rg_n * 64; idx += 128) {
      const int rr = idx >> 6, d = (idx & 63) * 2;
      float mm = -INFINITY;
#pragma unroll
      for (int w = 0; w < 4; ++w) mm = fmaxf(mm, cm_ml[(w * 16 + rr) * 2]);
      float a0f = 0.f, a1f = 0.f, ll = 0.f;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const float mw = cm_ml[(w * 16 + rr) * 2];
        if (mw == -INFINITY) continue;
        const float f = fast_exp2(mw - mm);
        a0f += f * cm_o[(w * 16 + rr) * 128 + d];
        a1f += f * cm_o[(w * 16 + rr) * 128 + d + 1];
        ll += f * cm_ml[(w * 16 + rr) * 2 + 1];
      }
      emit(rg + rr, d, a0f, a1f, mm, ll);
    }
    __syncthreads();
  }
}

// The protocol.  Call with ALL 128 threads after this CTA's partial has been stored to w.ws_o / w.ws_ml.
// emit_final(r, d, v0, v1, mm, ll): NORMALISED outputs of dims d, d+1 of row r (+ the merged max / row sum), called by
// the one CTA of the item that performs the final merge.  s_flag: one int of shared memory.
template <int ROWS, typename EmitFinal>
__device__ __forceinline__ void split_kv_finish(const SplitWs& w, long long item, int split, int splits, int rows,
                                                float* cm_o, float* cm_ml, int* s_flag, EmitFinal emit_final) {
  const int tid = threadIdx.x;
  const int ng = w.n_groups;
  int* cnt = w.counters + item * (1 + ng);
  const float* po = w.ws_o + item * splits * (long long)(ROWS * 128);
  const float* pml = w.ws_ml + item * splits * (long long)(ROWS * 2);
  auto final_emit = [&](int r, int d, float a0, float a1, float mm, float ll) {
    const float inv = ll > 0.f ? 1.f / ll : 0.f;
    emit_final(r, d, a0 * inv, a1 * inv, mm, ll);
  };
  __threadfence();
  __syncthreads();
  if (ng == 1) {
    if (tid == 0) *s_flag = (atomicAdd(&cnt[0], 1) == splits - 1);
    __syncthreads();
    if (!*s_flag) return;
    __threadfence();
    merge_partials_cta<ROWS>(po, pml, splits, rows, cm_o, cm_ml, final_emit);
    if (tid == 0) cnt[0] = 0;  // leave the workspace ready for the next launch
    return;
  }
  const int grp = split / kMergeGroup;
  const int gsz = min(kMergeGroup, splits - grp * kMergeGroup);
  if (tid == 0) *s_flag = (atomicAdd(&cnt[1 + grp], 1) == gsz - 1);
  __syncthreads();
  if (!*s_flag) return;
  __threadfence();
  float* go = w.g_o + (item * ng + grp) * (long long)(ROWS * 128);
  float* gml = w.g_ml + (item * ng + grp) * (long long)(ROWS * 2);
  merge_partials_cta<ROWS>(po + (long long)grp * kMergeGroup * (ROWS * 128), pml + (long long)grp * kMergeGroup * (ROWS * 2),
                           gsz, rows, cm_o, cm_ml, [&](int r, int d, float a0, float a1, float mm, float ll) {
                             *reinterpret_cast<float2*>(&go[r * 128 + d]) = make_float2(a0, a1);
                             if (d == 0) {
                               gml[r * 2] = mm;
                               gml[r * 2 + 1] = ll;
                             }
                           });
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    cnt[1 + grp] = 0;
    *s_flag = (atomicAdd(&cnt[0], 1) == ng - 1);
  }
  __syncthreads();
  if (!*s_flag) return;
  __threadfence();
  merge_partials_cta<ROWS>(w.g_o + item * ng * (long long)(ROWS * 128), w.g_ml + item * ng * (long long)(ROWS * 2), ng, rows,
                           cm_o, cm_ml, final_emit);
  if (tid == 0) cnt[0] = 0;
}

// ---------------------------------------------------------------------------------------------
// per-DEVICE launch attributes (one process may drive several GPUs, as the reference's tensor_parallel mode does,
// duo_attn/utils.py:206-227: cudaFuncSetAttribute is per device, so the "already set" memo is a device bit mask)
// ---------------------------------------------------------------------------------------------
int sm_count_current_device();  // api.cu
// Bytes kept free for a kernel's static __shared__ arrays when a launcher decides whether its dynamic shared memory
// still fits the 48 KB a launch gets without cudaFuncAttributeMaxDynamicSharedMemorySize (the row-norm kernels use
// well under 1 KB of static shared memory).
constexpr size_t kStaticSmemHeadroom = 1024;
template <typename K>
inline int ensure_dyn_smem(K kern, int bytes, unsigned long long* done_mask, bool max_carveout = false) {
  int dev = 0;
  DUO_CUDA_TRY(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (__atomic_load_n(done_mask, __ATOMIC_ACQUIRE) & bit) return DUO_OK;
  DUO_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  if (max_carveout)
    DUO_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  __atomic_fetch_or(done_mask, bit, __ATOMIC_RELEASE);
  return DUO_OK;
}

// ---------------------------------------------------------------------------------------------
// launch planning shared by the bandwidth launchers (attn_mma.cu, attn_int4.cu)
// ---------------------------------------------------------------------------------------------
// Keys per split when `nkeys` keys are cut into `splits` pieces: whole `tile`-key tiles, at least one.  The kernels
// recompute it from the device copy of the cache state on CUDA-graph replay.
__host__ __device__ __forceinline__ long long split_keys(long long nkeys, long long splits, int tile) {
  long long kps = (nkeys + splits - 1) / splits;
  kps = (kps + tile - 1) / tile * tile;
  return kps < tile ? tile : kps;
}

// Sequence-sharded caches (duo_attention_seq, duo_attention_seq_int4): position p lives on rank (p / block) % world, in
// local row (p / (block * world)) * block + p % block.  Rows of `rank`'s slice that hold positions < n (host twin:
// seqshard.SeqShardPlan.local_len).
__host__ __device__ __forceinline__ long long seq_local_len(long long n, int rank, int world, int block) {
  const long long round = (long long)block * world;
  const long long full_rounds = n / round, rem = n % round;
  long long extra = rem - (long long)rank * block;
  extra = extra < 0 ? 0 : (extra > block ? block : extra);
  return full_rounds * block + extra;
}

// Splits per retrieval item that bring the grid to `budget` CTAs next to `stream_ctas` streaming CTAs.
__host__ __device__ inline int split_want(int budget, int full_ctas, int stream_ctas) {
  const int want = (budget - stream_ctas > 0 ? budget - stream_ctas : 1) / full_ctas;
  return want < 1 ? 1 : want;
}

struct SplitPlan {
  int splits;
  long long keys_per_split;
};

// The split-KV policy: the retrieval items (`full_ctas` CTAs before splitting) split their `nkeys` keys so that the
// grid fills `budget` CTAs (k per SM, k = the kernel's occupancy), with at least `min_keys` keys per split and at most
// 512 splits.  A split is a whole number of `tile`-key tiles, so fewer splits may end up covering the keys.
inline SplitPlan plan_splits(long long nkeys, int budget, int full_ctas, int stream_ctas, int tile, int min_keys) {
  long long splits = 1;
  if (full_ctas > 0) {
    const long long max_by_len = (nkeys + min_keys - 1) / min_keys;
    splits = std::min<long long>({split_want(budget, full_ctas, stream_ctas), std::max(1LL, max_by_len), 512});
  }
  const long long kps = split_keys(nkeys, splits, tile);
  splits = (nkeys + kps - 1) / kps;
  return {(int)std::max(1LL, splits), kps};
}

// ---- ragged decode batches (duo_decode_ragged, duo_decode_ragged_int4) ------------------------------------------
// Keys per split of a ragged decode batch.  Chosen from the mean row length so that, with every row at the same
// length, it equals plan_splits' partition (>= min_keys keys per split, <= want and <= 512 splits, whole `tile`-key
// tiles), and raised so that no row needs more than 512 splits.  Row b then takes max(1, ceil(len_b / kps)) splits.
// Host twin: kv_cache.ragged_partition.
__host__ __device__ __forceinline__ long long ragged_keys_per_split(long long n_sum, long long n_max, int batch,
                                                                    int want, int tile, int min_keys) {
  const long long lbar = (n_sum + batch - 1) / batch;
  long long s = (lbar + min_keys - 1) / min_keys;
  if (s < 1) s = 1;
  if (s > want) s = want;
  if (s > 512) s = 512;
  const long long kps = split_keys(lbar, s, tile);
  const long long cap = ((n_max + 511) / 512 + tile - 1) / tile * tile;
  return kps < cap ? cap : kps;
}

// row_state[b][3] is a flags word.  Bit 0 set: row b is IDLE and sits out every batched launch of its cache (no read of
// its keys or ring, no write, no row_state change); the other bits are 0.  The active rows are partitioned as a compact
// batch of just those rows would be.  Host twin: kv_cache.ragged_partition(..., active=).
__host__ __device__ __forceinline__ bool ragged_idle(const long long* rs, int b) { return (rs[4 * b + 3] & 1) != 0; }

// Split budget per (row, retrieval head) of a ragged batch of `batch` rows at `budget` CTAs (ragged_geom's `want`).
__host__ __device__ inline int ragged_want(int batch, int n_full, int n_stream, int budget) {
  const int want = split_want(budget, batch * (n_full > 1 ? n_full : 1), batch * n_stream);
  return want < 512 ? want : 512;
}

// The split budget of a launch with n_act active rows out of p.batch: the launch's own p.rg_want when every row is
// active, else the compact batch's, clamped to floor(rg_slots / n_act) - 1 so that its splits fit the launch's grid.
template <typename P>
__device__ __forceinline__ int ragged_active_want(const P& p, int n_act) {
  if (n_act == p.batch) return p.rg_want;
  const int want = ragged_want(n_act, p.n_full, p.n_stream, p.rg_budget), fit = p.rg_slots / n_act - 1;
  return want < fit ? want : fit;
}

// Keys per split of the active rows of a batch whose row r has len_of(r) keys (the shared-prefix decode: a row's own
// keys); rs: the [batch][4] row_state array.
template <typename Len, typename P>
__device__ __forceinline__ long long ragged_batch_kps_of(Len len_of, const long long* rs, const P& p, int tile,
                                                         int min_keys) {
  long long n_sum = 0, n_max = 0;
  int n_act = 0;
  for (int r = 0; r < p.batch; ++r) {
    if (ragged_idle(rs, r)) continue;
    const long long len = len_of(r);
    ++n_act;
    n_sum += len;
    n_max = len > n_max ? len : n_max;
  }
  if (n_act == 0) return tile;  // every row idle: no slot is taken
  return ragged_keys_per_split(n_sum, n_max, n_act, ragged_active_want(p, n_act), tile, min_keys);
}

// Keys per split of the batch in device memory: row b has rs[4 b] + q_add keys.
template <typename P>
__device__ __forceinline__ long long ragged_batch_kps(const long long* rs, const P& p, int q_add, int tile,
                                                      int min_keys) {
  return ragged_batch_kps_of([&](int r) { return rs[4 * r] + q_add; }, rs, p, tile, min_keys);
}

// Where grid slot `c` of a retrieval head falls: active row b's splits occupy consecutive slots from slot_base, an idle
// row takes none.  b == batch: an idle slot (the batch needs fewer splits than the grid holds).
struct RaggedSlot {
  int b, split, splits;
  long long slot_base;
};
// ragged_slot for a batch whose row r has len_of(r) keys.
template <typename Len>
__device__ __forceinline__ RaggedSlot ragged_slot_of(Len len_of, const long long* rs, int batch, long long kps, int c) {
  RaggedSlot s;
  s.slot_base = 0;
  s.splits = 0;
  for (s.b = 0; s.b < batch; ++s.b) {
    if (ragged_idle(rs, s.b)) continue;
    const long long len = len_of(s.b);
    s.splits = len > kps ? (int)((len + kps - 1) / kps) : 1;
    if (c < s.slot_base + s.splits) break;
    s.slot_base += s.splits;
  }
  s.split = c - (int)s.slot_base;
  return s;
}
__device__ __forceinline__ RaggedSlot ragged_slot(const long long* rs, int batch, int q_add, long long kps, int c) {
  return ragged_slot_of([&](int r) { return rs[4 * r] + q_add; }, rs, batch, kps, c);
}

// Points `w` (carved by the ragged geometry's layout) at the slice of (row b, retrieval head kvh): its own counters
// and level-2 partials, its level-1 partials at the row's grid slots.  The kernel then uses item 0.
template <int ROWS>
__device__ __forceinline__ void ragged_ws_slice(SplitWs& w, int b, int kvh, int n_full, int rg_slots,
                                                const RaggedSlot& s) {
  const long long item = (long long)b * n_full + kvh, ngm = w.n_groups;
  const long long part = (long long)kvh * rg_slots + s.slot_base;
  w.counters += item * (1 + ngm);
  w.ws_ml += part * (ROWS * 2);
  w.ws_o += part * (ROWS * 128);
  w.g_ml += item * ngm * (ROWS * 2);
  w.g_o += item * ngm * (ROWS * 128);
  w.n_groups = s.splits <= kMergeGroup ? 1 : (s.splits + kMergeGroup - 1) / kMergeGroup;
}

// Grid geometry of a ragged launch.  It depends only on the layer and the device, never on the row lengths, so a
// captured graph stays valid while the rows grow.  `want` is plan_splits' split budget per (row, retrieval head) at
// `ctas_per_sm` CTAs per SM; with kps from ragged_keys_per_split, sum_b ceil(len_b / kps) <= batch * want + batch, so
// batch * (want + 1) slots per retrieval head always suffice.  `rows`: query rows per partial.  `budget` is the CTA
// budget the kernels re-plan the active rows with when some rows are idle (ragged_active_want).
struct RaggedGeom {
  int want, slots, budget;
  SplitWsLayout ws;  // `slots` partials per retrieval head; level-2 groups for the most splits a row can take
  size_t ws_bytes;   // SIZE_MAX if the counters do not fit
};

inline RaggedGeom ragged_geom(int batch, int n_full, int n_stream, int sm_count, int ctas_per_sm, int rows) {
  RaggedGeom g{};
  g.budget = ctas_per_sm * sm_count;
  g.want = ragged_want(batch, n_full, n_stream, g.budget);
  g.slots = batch * (g.want + 1);
  const long long items = (long long)batch * n_full;
  const int ng_max = split_groups(std::min(512, g.slots));
  g.ws = {items, ng_max, (long long)n_full * g.slots, items * ng_max, rows};
  g.ws_bytes = n_full > 0 ? split_ws_bytes(g.ws) : 0;
  return g;
}

// Workspace of a ragged launch for any split of n_kv heads into retrieval and streaming heads, on this device.
inline size_t ragged_ws_need(int batch, int n_kv, int ctas_per_sm, int rows) {
  const int sms = sm_count_current_device();
  size_t need = 0;
  for (int nf = 1; nf <= n_kv; ++nf) {
    const size_t b = ragged_geom(batch, nf, n_kv - nf, sms, ctas_per_sm, rows).ws_bytes;
    if (b == (size_t)-1) return b;
    need = std::max(need, b);
  }
  return need;
}

// ---- batched ragged prefill (duo_prefill_ragged) ------------------------------------------------------------------
// Row b of a ragged batch takes a chunk of len[b] >= 0 tokens; the chunks are packed back to back, row b's first token
// at packed index off[b] (off[batch] = the packed tokens T).  The host copies the table into the kernel parameters of
// the three launches (append, attention, commit), which read each row's occupancy from row_state, its region
// {first, cap} from row_geom (pooled layers, else NULL) and its {donor, P} from row_share (NULL: nothing shared).
struct RaggedChunks {
  const long long* row_state;
  const long long* row_geom;
  const long long* row_share;
  int batch;
  int len[DUO_RAGGED_MAX_BATCH];
  int off[DUO_RAGGED_MAX_BATCH + 1];
};

// The row whose chunk holds packed token `tok` (< off[batch]): the last row b with off[b] <= tok, which has len > 0.
__device__ __forceinline__ int ragged_chunk_row(const RaggedChunks& rc, long long tok) {
  int lo = 0, hi = rc.batch;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (rc.off[mid] <= tok) lo = mid; else hi = mid;
  }
  return lo;
}

// Keys [0, P) of a row that shares its donor's prefix are the donor's region rows; 0 for every other row (a donor's own
// entry names itself).
__device__ __forceinline__ long long ragged_chunk_share(const RaggedChunks& rc, int b, int& donor) {
  donor = rc.row_share ? (int)rc.row_share[2 * b] : -1;
  if (donor < 0 || donor == b) return 0;
  return rc.row_share[2 * b + 1];
}

// Pool row of key row j of retrieval head h in row b's region: row b's region holds [n_full][cap] rows from pool row
// first * n_full (kv_cache.pool_layout).
__device__ __forceinline__ long long ragged_pool_row(const RaggedChunks& rc, int b, int n_full, int h, long long j) {
  const long long first = rc.row_geom[2 * b], cap = rc.row_geom[2 * b + 1];
  return first * n_full + (long long)h * cap + j;
}

// ---- shared prefixes (duo_decode_ragged_shared, both KV formats) ------------------------------------------------
// The key tile of both prefix kernels (attn_mma.cu's 64-row variant and duo_attn_int4_kernel<1>).
constexpr int kSharePrefixTile = 64;

// Keys row b shares with its donor (row_share {d, P}): P, or 0 for a row that shares nothing.
__device__ __forceinline__ long long share_keys(const long long* rsh, int b) { return rsh[2 * b] >= 0 ? rsh[2 * b + 1] : 0; }

// Row b's place among the active rows that share one prefix {d, P} (P > 0): lead = the lowest such row, rank = b's index
// among them in row order, cnt = their number when b leads them (else 0).  lead = -1 for a row that shares nothing or is
// idle (rs: row_state, ragged_idle); a group whose members are all idle has no lead, an idle donor's group is led by its
// lowest active sharer.
__device__ __forceinline__ void share_rank(const long long* rsh, const long long* rs, int batch, int b, int& lead,
                                           int& rank, int& cnt) {
  const long long d = rsh[2 * b], P = rsh[2 * b + 1];
  lead = -1;
  rank = cnt = 0;
  if (d < 0 || P <= 0 || ragged_idle(rs, b)) return;
  lead = b;
  int after = 0;
  for (int r = 0; r < batch; ++r) {
    if (r == b || rsh[2 * r] != d || rsh[2 * r + 1] != P || ragged_idle(rs, r)) continue;
    if (r < b) {
      if (lead == b) lead = r;
      ++rank;
    } else {
      ++after;
    }
  }
  cnt = lead == b ? 1 + after : 0;
}

// The prefix kernel's work item at grid slot c of a retrieval head (one thread).  The groups of rows sharing one
// prefix, in the order of their lead rows, are cut into blocks of 64 packed rows (rpm per row); every block is an item
// and takes ceil(P / kps) consecutive slots.  kps >= 256 keys comes from the items' total keys over the slots they may
// use, raised so that no item takes more than max_splits.  Since rpm <= 16 there are at most `batch` items, and the
// slots (budget + batch) always suffice.  out = {lead, block, split, splits, kps, slot_base, item, members}; lead = -1:
// an idle slot.
static __device__ __noinline__ void share_prefix_slot(const long long* rsh, const int* s_lead, const int* s_cnt, int batch,
                                               int rpm, int slots, int max_splits, int c, long long* out) {
  long long total = 0, pmax = 0;
  int n_items = 0;
  for (int b = 0; b < batch; ++b) {
    if (s_lead[b] != b) continue;
    const int nb = (s_cnt[b] * rpm + 63) / 64;
    n_items += nb;
    total += nb * rsh[2 * b + 1];
    pmax = max(pmax, rsh[2 * b + 1]);
  }
  out[0] = -1;
  if (n_items == 0) return;
  long long kps = max(split_keys(total, slots - n_items, kSharePrefixTile), (long long)(4 * kSharePrefixTile));
  kps = max(kps, ((pmax + max_splits - 1) / max_splits + kSharePrefixTile - 1) / kSharePrefixTile * kSharePrefixTile);
  long long base = 0;
  int item = 0;
  for (int b = 0; b < batch; ++b) {
    if (s_lead[b] != b) continue;
    const long long P = rsh[2 * b + 1];
    const int nb = (s_cnt[b] * rpm + 63) / 64, sp = (int)((P + kps - 1) / kps);
    for (int k = 0; k < nb; ++k, ++item, base += sp) {
      if (c < base + sp) {
        const long long v[8] = {b, k, c - base, sp, kps, base, item, s_cnt[b]};
        for (int i = 0; i < 8; ++i) out[i] = v[i];
        return;
      }
    }
  }
}
// Grid of the prefix kernel: per retrieval head, the ~2 CTAs/SM budget plus one slot per row (a batch never has more
// items than rows, see share_prefix_slot).  The most splits one item may take keeps the items' arrival counters inside
// the fixed counter region.  Like ragged_geom, it depends only on the layer and the device.
struct PrefixGeom {
  int slots, max_splits;
  SplitWsLayout ws;
  size_t ws_bytes;  // SIZE_MAX if the counters do not fit
};
inline PrefixGeom prefix_geom(int batch, int n_full, int sm_count) {
  PrefixGeom g{};
  const long long items = (long long)batch * std::max(n_full, 1);
  const long long ng_cap = (long long)(kSplitCounterBytes / 4) / items - 1;
  g.max_splits = (int)std::min<long long>(512, 16 * std::max<long long>(ng_cap, 1));
  g.slots = std::max(1, 2 * sm_count / std::max(n_full, 1)) + batch;
  const int ng = split_groups(std::min(g.max_splits, g.slots));
  g.ws = {items, ng, (long long)n_full * g.slots, ng > 1 ? items * ng : 0, 64};
  g.ws_bytes = n_full > 0 ? split_ws_bytes(g.ws) : 0;
  return g;
}

// The workspace of the cascade: the two launches run one after the other, so their split partials share one region
// (and the counter region, which each launch leaves zeroed); the prefix partials, which the suffix launch reads, follow
// it: [batch][q_len][n_q_heads] rows of 128 fp32 O, then as many fp32 lse.
inline size_t shared_split_bytes(const RaggedGeom& g, const PrefixGeom& pg) {
  if (g.ws_bytes == (size_t)-1 || pg.ws_bytes == (size_t)-1) return (size_t)-1;
  return (std::max(g.ws_bytes, pg.ws_bytes) + 255) / 256 * 256;
}

// Fills the fields AttnParams (attn_mma.cu) and I4Params (attn_int4.cu) share: addressing of a q_len-token chunk of
// q rows `q_row_stride` elements apart, the layer's head geometry and the cache occupancy `st`.
template <typename P>
inline void fill_common_params(P& p, const duo_layer_desc& d, const duo_cache_state& st, const void* q,
                               long long q_row_stride, void* out, int q_len, float scale) {
  const int n_q = (d.n_full + d.n_stream) * d.group;
  p.q = q;
  p.out = out;
  p.q_tok_stride = q_row_stride;
  p.q_batch_stride = q_row_stride * q_len;
  p.out_batch_stride = (long long)q_len * n_q * kHeadDim;
  p.q_len = q_len;
  p.n_q_heads = n_q;
  p.group = d.group;
  p.n_full = d.n_full;
  p.n_stream = d.n_stream;
  p.batch = d.batch;
  p.sink = d.sink;
  p.recent = d.recent;
  p.W = d.sink + d.recent;
  p.full_len = st.full_len;
  p.total = st.total;
  p.lo = st.lo;
  p.dstate = reinterpret_cast<const long long*>(st.device_state);
  p.scale_log2 = scale * 1.4426950408889634f;
  // streaming cache scan range: slots [0, min(W, total)) can hold live tokens
  p.cache_scan = (int)std::min<long long>(p.W, st.total);
}

struct FusedArgs {  // one-launch decode step (duo_decode_fused): q points at the raw qkv rows
  const void* cos = nullptr;
  const void* sin = nullptr;
  int rope_mode = DUO_ROPE_NONE;
};

// The RoPE tables and the offsets of the k / v sections inside a qkv row; after fill_common_params.
template <typename P>
inline void fill_fused_args(P& p, const FusedArgs& fa) {
  p.cos = fa.cos;
  p.sin = fa.sin;
  p.rope_mode = fa.rope_mode;
  p.k_off = (long long)p.n_q_heads * kHeadDim;
  p.v_off = (long long)(p.n_q_heads + p.n_full + p.n_stream) * kHeadDim;
}

// The four K/V maps (64- or 128-row boxes) of a layer, as the kernels take them.  A layer without retrieval (or
// without streaming) heads still needs some valid descriptor in that parameter slot: the other class's map stands
// in; it is never dereferenced because no CTA of that class is launched.
struct KvMaps {
  const CUtensorMap *fk, *fv, *rk, *rv;
};
inline KvMaps kv_maps(const duo_layer* L, bool box128) {
  const LayerMaps& m = L->maps;
  const CUtensorMap* fk = box128 ? &m.full_k128 : &m.full_k64;
  const CUtensorMap* fv = box128 ? &m.full_v128 : &m.full_v64;
  const CUtensorMap* rk = box128 ? &m.ring_k128 : &m.ring_k64;
  const CUtensorMap* rv = box128 ? &m.ring_v128 : &m.ring_v64;
  return {L->has_full_maps ? fk : rk, L->has_full_maps ? fv : rv, L->has_ring_maps ? rk : fk,
          L->has_ring_maps ? rv : fv};
}

// f(T{}) with T the layer's 16-bit activation type
template <typename F>
inline int dispatch_dtype(int dtype, F&& f) {
  if (dtype == DUO_DT_BF16) return f(__nv_bfloat16{});
  return f(__half{});
}

}  // namespace duo
