// One-shot all-reduce over NVLink peer memory FUSED with the residual add + RMSNorm that follows it
// (SURVEY.md §8e "custom one-shot kernel", §8f3 "fuse o_proj + all-reduce + residual + RMSNorm").
//
// Head-parallel TP leaves a row-parallel partial of the o_proj (and down_proj) output on every rank; the reference
// sums them through tensor_parallel's "sum" output rule (duo_attn/utils.py:174-176).  At decode that is an 8 KB
// exchange: pure latency.  NCCL costs ~15 us per call (64 calls per step); this kernel does the exchange, the sum,
// the residual add and the next RMSNorm in ONE launch per site:
//
//   1. push : every rank stores its partial row into slot [epoch&1][rank] of EVERY rank's receive buffer (plain 16 B
//             stores through the peer mapping: posted writes, no read round trip over NVLink);
//   2. flag : bar.sync, then W threads fence.sys and st.release.sys the epoch into the W receivers' flag words;
//   3. wait : W threads spin (ld.acquire.sys) on the local flag words until every sender's epoch has arrived;
//   4. sum  : all ranks add the W rows in the SAME order (rank 0..W-1, fp32) -> bit-identical residual streams on every
//             rank; rounded to the activation dtype (as an all-reduce result would be), + residual, RMSNorm.
//
// Epochs live in device memory and only ever increase, so the kernel is CUDA-graph replayable; the receive buffer is
// double-buffered by epoch parity (a rank can be at most one call ahead of the slowest peer: to finish call k+1 it
// needs every peer's k+1 flag, which a peer only sends after it has finished reading call k).  One CTA per row, rows
// <= max_rows (decode and small chunks; large prefill chunks are bandwidth-bound and stay on NCCL).
//
//
// The same push / flag / wait primitive carries the exchange step of the sequence-sharded decode (seq_merge_kernel
// below): (O, log-sum-exp) partials of the retrieval heads instead of hidden-state rows.
#include "duo_common.cuh"

struct duo_comm {
  duo_comm_desc d;
};
struct duo_seqcomm {
  duo_seqcomm_desc d;
};

namespace duo {

constexpr int kMaxWorld = 8;
constexpr int kCommThreads = 512;

struct CommParams {
  void* peer_data[kMaxWorld];
  unsigned int* peer_flags[kMaxWorld];
  const void* partial;
  const void* residual;
  const void* weight;
  void* out_norm;
  void* out_res;
  int* state;  // [max_rows] epochs | [1] error word
  int rank, world, hidden, max_rows;
  float eps;
};

template <typename T>
struct CmCvt;
template <>
struct CmCvt<__nv_bfloat16> {
  __device__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <>
struct CmCvt<__half> {
  __device__ static float to_f(__half v) { return __half2float(v); }
  __device__ static __half from_f(float v) { return __float2half_rn(v); }
};
template <typename T>
struct alignas(16) CmVec8 {
  T v[8];
};

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

template <typename T>
__global__ void __launch_bounds__(kCommThreads) ar_add_rmsnorm_kernel(const CommParams p) {
  extern __shared__ float s_row[];  // hidden floats: the summed row, already rounded to T
  __shared__ float s_part[kCommThreads / 32];
  __shared__ int s_epoch;
  const int row = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) s_epoch = p.state[row] + 1;
  __syncthreads();
  const unsigned int epoch = (unsigned int)s_epoch;
  const int slot = (int)(epoch & 1u);
  const int hidden = p.hidden;

  // ---- 1. push my partial row to every rank (including myself) --------------------------------------------
  {
    const T* src = reinterpret_cast<const T*>(p.partial) + (long long)row * hidden;
    const long long dst_off = (((long long)slot * p.world + p.rank) * p.max_rows + row) * hidden;
    for (int i = tid * 8; i < hidden; i += kCommThreads * 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(src + i);
#pragma unroll
      for (int q = 0; q < kMaxWorld; ++q) {
        if (q < p.world) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.peer_data[q]) + dst_off + i) = v;
      }
    }
  }
  __syncthreads();
  // ---- 2. publish: one thread per receiver ---------------------------------------------------------------------
  if (tid < p.world) {
    __threadfence_system();
    unsigned int* f = nullptr;
#pragma unroll
    for (int q = 0; q < kMaxWorld; ++q)
      if (q == tid) f = p.peer_flags[q];
    st_release_sys(f + (long long)row * p.world + p.rank, epoch);
  }
  // ---- 3. wait for every sender's epoch (bounded: a lost peer sets the error word instead of hanging the GPU) -----
  if (tid < p.world) {
    unsigned int* mine = nullptr;
#pragma unroll
    for (int q = 0; q < kMaxWorld; ++q)
      if (q == p.rank) mine = p.peer_flags[q];
    const unsigned int* f = mine + (long long)row * p.world + tid;
    const long long t0 = clock64();
    while ((int)(ld_acquire_sys(f) - epoch) < 0) {
      if (clock64() - t0 > 6000000000LL) {  // ~3 s
        p.state[p.max_rows] = 1;
        break;
      }
    }
  }
  __syncthreads();
  // ---- 4. sum in rank order, residual add, RMSNorm (arithmetic of add_rmsnorm_kernel, elementwise.cu) -------------
  const T* my_data = nullptr;
#pragma unroll
  for (int q = 0; q < kMaxWorld; ++q)
    if (q == p.rank) my_data = reinterpret_cast<const T*>(p.peer_data[q]);
  const T* rr = p.residual ? reinterpret_cast<const T*>(p.residual) + (long long)row * hidden : nullptr;
  T* out_res = p.out_res ? reinterpret_cast<T*>(p.out_res) + (long long)row * hidden : nullptr;
  float ss = 0.f;
  for (int i = tid * 8; i < hidden; i += kCommThreads * 8) {
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int s = 0; s < p.world; ++s) {
      const long long off = (((long long)slot * p.world + s) * p.max_rows + row) * hidden + i;
      const uint4 raw = __ldcg(reinterpret_cast<const uint4*>(my_data + off));  // L2: peers wrote it over NVLink
      const CmVec8<T> v = *reinterpret_cast<const CmVec8<T>*>(&raw);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += CmCvt<T>::to_f(v.v[k]);
    }
    CmVec8<T> a;
#pragma unroll
    for (int k = 0; k < 8; ++k) a.v[k] = CmCvt<T>::from_f(acc[k]);
    if (rr) {
      const CmVec8<T> b = *reinterpret_cast<const CmVec8<T>*>(rr + i);
#pragma unroll
      for (int k = 0; k < 8; ++k) a.v[k] = CmCvt<T>::from_f(CmCvt<T>::to_f(b.v[k]) + CmCvt<T>::to_f(a.v[k]));
    }
    if (out_res) *reinterpret_cast<CmVec8<T>*>(out_res + i) = a;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float f = CmCvt<T>::to_f(a.v[k]);
      s_row[i + k] = f;
      ss += f * f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((tid & 31) == 0) s_part[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < kCommThreads / 32; ++w) tot += s_part[w];
  const float inv = rsqrtf(tot / (float)hidden + p.eps);
  const T* weight = reinterpret_cast<const T*>(p.weight);
  T* out_norm = reinterpret_cast<T*>(p.out_norm) + (long long)row * hidden;
  for (int i = tid * 8; i < hidden; i += kCommThreads * 8) {
    const CmVec8<T> w = *reinterpret_cast<const CmVec8<T>*>(weight + i);
    CmVec8<T> o;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const T n = CmCvt<T>::from_f(s_row[i + k] * inv);
      o.v[k] = CmCvt<T>::from_f(CmCvt<T>::to_f(w.v[k]) * CmCvt<T>::to_f(n));
    }
    *reinterpret_cast<CmVec8<T>*>(out_norm + i) = o;
  }
  if (tid == 0) p.state[row] = (int)epoch;
}

// ---------------------------------------------------------------------------------------------------------------
// Sequence-sharded decode: exchange + merge of the retrieval heads' partial attention.  One CTA of 128 threads per
// (token, retrieval q-head) row; payload per row and sender = 128 fp32 outputs + the log-sum-exp, padded to 132 floats.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kSeqRowFloats = 132;

struct SeqMergeParams {
  float* peer_data[kMaxWorld];
  unsigned int* peer_flags[kMaxWorld];
  const float* part_o;
  const float* part_lse;
  void* out;
  int* state;
  int rank, world, max_rows, heads_total, heads_used;
};

template <typename T>
__global__ void __launch_bounds__(128) seq_merge_kernel(const SeqMergeParams p) {
  __shared__ int s_epoch;
  __shared__ float s_w[kMaxWorld];
  const int row = blockIdx.x, tid = threadIdx.x;
  const int tok = row / p.heads_used, h = row % p.heads_used;
  const long long src_row = (long long)tok * p.heads_total + h;
  if (tid == 0) s_epoch = p.state[row] + 1;
  __syncthreads();
  const unsigned int epoch = (unsigned int)s_epoch;
  const int slot = (int)(epoch & 1u);
  // ---- 1. push my partial row to every rank (posted 4-byte stores, 512 B coalesced per peer) -------------------
  {
    const float v = p.part_o[src_row * kHeadDim + tid];
    const float l = p.part_lse[src_row];
    const long long off = (((long long)slot * p.world + p.rank) * p.max_rows + row) * kSeqRowFloats;
#pragma unroll
    for (int q = 0; q < kMaxWorld; ++q) {
      if (q < p.world) {
        p.peer_data[q][off + tid] = v;
        if (tid == 0) p.peer_data[q][off + kHeadDim] = l;
      }
    }
  }
  __syncthreads();
  // ---- 2. publish / 3. wait (bounded) ----------------------------------------------------------------------------
  if (tid < p.world) {
    __threadfence_system();
    unsigned int* f = nullptr;
#pragma unroll
    for (int q = 0; q < kMaxWorld; ++q)
      if (q == tid) f = p.peer_flags[q];
    st_release_sys(f + (long long)row * p.world + p.rank, epoch);
    unsigned int* mine = nullptr;
#pragma unroll
    for (int q = 0; q < kMaxWorld; ++q)
      if (q == p.rank) mine = p.peer_flags[q];
    const unsigned int* w = mine + (long long)row * p.world + tid;
    const long long t0 = clock64();
    while ((int)(ld_acquire_sys(w) - epoch) < 0) {
      if (clock64() - t0 > 6000000000LL) {  // ~3 s
        p.state[p.max_rows] = 1;
        break;
      }
    }
  }
  __syncthreads();
  // ---- 4. merge the `world` partials in rank order: out = sum_s 2^(lse_s - max) o_s / sum_s 2^(lse_s - max) -----------
  const float* my_data = nullptr;
#pragma unroll
  for (int q = 0; q < kMaxWorld; ++q)
    if (q == p.rank) my_data = p.peer_data[q];
  const float* base = my_data + ((long long)slot * p.world * p.max_rows + row) * kSeqRowFloats;
  const long long sstride = (long long)p.max_rows * kSeqRowFloats;
  if (tid < p.world) s_w[tid] = __ldcg(base + tid * sstride + kHeadDim);
  __syncthreads();
  float mx = -INFINITY;
  for (int s2 = 0; s2 < p.world; ++s2) mx = fmaxf(mx, s_w[s2]);
  float acc = 0.f, wsum = 0.f;
  for (int s2 = 0; s2 < p.world; ++s2) {
    const float l = s_w[s2];
    if (l == -INFINITY) continue;
    const float w = fast_exp2(l - mx);
    acc += w * __ldcg(base + s2 * sstride + tid);
    wsum += w;
  }
  const float v = wsum > 0.f ? acc / wsum : 0.f;
  reinterpret_cast<T*>(p.out)[src_row * kHeadDim + tid] = CmCvt<T>::from_f(v);
  if (tid == 0) p.state[row] = (int)epoch;
}

static size_t elt_bytes(int dtype) { return (dtype == DUO_DT_BF16 || dtype == DUO_DT_FP16) ? 2 : 0; }

}  // namespace duo

extern "C" {

size_t duo_comm_data_bytes(int32_t world, int32_t hidden, int32_t max_rows, int32_t dtype) {
  if (world < 1 || hidden < 1 || max_rows < 1) return 0;
  return (size_t)2 * world * max_rows * hidden * duo::elt_bytes(dtype);
}

size_t duo_comm_flag_bytes(int32_t world, int32_t max_rows) {
  if (world < 1 || max_rows < 1) return 0;
  return ((size_t)world * max_rows * 4 + 255) / 256 * 256;
}

int duo_comm_create(const duo_comm_desc* desc, duo_comm** out) {
  if (!desc || !out) {
    duo::set_error("duo_comm_create: null argument");
    return DUO_EINVAL;
  }
  const duo_comm_desc& d = *desc;
  if (d.world < 2 || d.world > duo::kMaxWorld || d.rank < 0 || d.rank >= d.world || d.max_rows < 1 || d.max_rows > 64 ||
      d.hidden < 8 || d.hidden % 8 != 0 || d.hidden > 16384 || duo::elt_bytes(d.dtype) == 0 || !d.local_state) {
    duo::set_error("duo_comm_create: bad descriptor (world %d, rank %d, hidden %d, max_rows %d)", d.world, d.rank,
                   d.hidden, d.max_rows);
    return DUO_EINVAL;
  }
  for (int r = 0; r < d.world; ++r) {
    if (!d.data[r] || !d.flags[r] || (reinterpret_cast<uintptr_t>(d.data[r]) & 15) ||
        (reinterpret_cast<uintptr_t>(d.flags[r]) & 3)) {
      duo::set_error("duo_comm_create: peer buffer %d missing or misaligned", r);
      return DUO_EINVAL;
    }
  }
  duo_comm* c = new duo_comm;
  c->d = d;
  *out = c;
  return DUO_OK;
}

void duo_comm_destroy(duo_comm* comm) { delete comm; }

int duo_allreduce_add_rmsnorm(const duo_comm* comm, const void* partial, const void* residual, const void* weight,
                              void* out_norm, void* out_res, int32_t rows, float eps, void* stream) {
  if (!comm || rows < 0 || (rows > 0 && (!partial || !weight || !out_norm))) {
    duo::set_error("duo_allreduce_add_rmsnorm: bad argument");
    return DUO_EINVAL;
  }
  const duo_comm_desc& d = comm->d;
  if (rows > d.max_rows) {
    duo::set_error("duo_allreduce_add_rmsnorm: %d rows exceed the communicator's max_rows %d", rows, d.max_rows);
    return DUO_EOVERFLOW;
  }
  if (rows == 0) return DUO_OK;
  duo::CommParams p{};
  for (int r = 0; r < d.world; ++r) {
    p.peer_data[r] = d.data[r];
    p.peer_flags[r] = reinterpret_cast<unsigned int*>(d.flags[r]);
  }
  p.partial = partial;
  p.residual = residual;
  p.weight = weight;
  p.out_norm = out_norm;
  p.out_res = out_res;
  p.state = reinterpret_cast<int*>(d.local_state);
  p.rank = d.rank;
  p.world = d.world;
  p.hidden = d.hidden;
  p.max_rows = d.max_rows;
  p.eps = eps;
  const size_t smem = (size_t)d.hidden * sizeof(float);
  cudaStream_t s = (cudaStream_t)stream;
  // the 48 KB default limit covers dynamic + static shared memory (s_part, s_epoch): hidden 12288 already needs the
  // opt-in
  const bool opt_in = smem + duo::kStaticSmemHeadroom > 48 * 1024;
  if (d.dtype == DUO_DT_BF16) {
    static unsigned long long attr_mask = 0;
    if (opt_in)
      if (int rc = duo::ensure_dyn_smem(duo::ar_add_rmsnorm_kernel<__nv_bfloat16>, 64 * 1024, &attr_mask)) return rc;
    duo::ar_add_rmsnorm_kernel<__nv_bfloat16><<<rows, duo::kCommThreads, smem, s>>>(p);
  } else {
    static unsigned long long attr_mask = 0;
    if (opt_in)
      if (int rc = duo::ensure_dyn_smem(duo::ar_add_rmsnorm_kernel<__half>, 64 * 1024, &attr_mask)) return rc;
    duo::ar_add_rmsnorm_kernel<__half><<<rows, duo::kCommThreads, smem, s>>>(p);
  }
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

size_t duo_seqcomm_data_bytes(int32_t world, int32_t max_rows) {
  if (world < 1 || max_rows < 1) return 0;
  return (size_t)2 * world * max_rows * duo::kSeqRowFloats * sizeof(float);
}

size_t duo_seqcomm_flag_bytes(int32_t world, int32_t max_rows) { return duo_comm_flag_bytes(world, max_rows); }

int duo_seqcomm_create(const duo_seqcomm_desc* desc, duo_seqcomm** out) {
  if (!desc || !out) {
    duo::set_error("duo_seqcomm_create: null argument");
    return DUO_EINVAL;
  }
  const duo_seqcomm_desc& d = *desc;
  if (d.world < 2 || d.world > duo::kMaxWorld || d.rank < 0 || d.rank >= d.world || d.max_rows < 1 || d.max_rows > 512 ||
      !d.local_state) {
    duo::set_error("duo_seqcomm_create: bad descriptor (world %d, rank %d, max_rows %d)", d.world, d.rank, d.max_rows);
    return DUO_EINVAL;
  }
  for (int r = 0; r < d.world; ++r) {
    if (!d.data[r] || !d.flags[r] || (reinterpret_cast<uintptr_t>(d.data[r]) & 15) ||
        (reinterpret_cast<uintptr_t>(d.flags[r]) & 3)) {
      duo::set_error("duo_seqcomm_create: peer buffer %d missing or misaligned", r);
      return DUO_EINVAL;
    }
  }
  duo_seqcomm* c = new duo_seqcomm;
  c->d = d;
  *out = c;
  return DUO_OK;
}

void duo_seqcomm_destroy(duo_seqcomm* comm) { delete comm; }

int duo_seq_merge(const duo_seqcomm* comm, const float* part_o, const float* part_lse, void* out, int32_t tokens,
                  int32_t heads_total, int32_t heads_used, int32_t dtype, void* stream) {
  if (!comm || tokens < 0 || heads_total < 1 || heads_used < 0 || heads_used > heads_total ||
      (dtype != DUO_DT_BF16 && dtype != DUO_DT_FP16)) {
    duo::set_error("duo_seq_merge: bad argument");
    return DUO_EINVAL;
  }
  const int rows = tokens * heads_used;
  if (rows == 0) return DUO_OK;
  if (!part_o || !part_lse || !out) {
    duo::set_error("duo_seq_merge: null buffer");
    return DUO_EINVAL;
  }
  const duo_seqcomm_desc& d = comm->d;
  if (rows > d.max_rows) {
    duo::set_error("duo_seq_merge: %d rows exceed the communicator's max_rows %d", rows, d.max_rows);
    return DUO_EOVERFLOW;
  }
  duo::SeqMergeParams p{};
  for (int r = 0; r < d.world; ++r) {
    p.peer_data[r] = reinterpret_cast<float*>(d.data[r]);
    p.peer_flags[r] = reinterpret_cast<unsigned int*>(d.flags[r]);
  }
  p.part_o = part_o;
  p.part_lse = part_lse;
  p.out = out;
  p.state = reinterpret_cast<int*>(d.local_state);
  p.rank = d.rank;
  p.world = d.world;
  p.max_rows = d.max_rows;
  p.heads_total = heads_total;
  p.heads_used = heads_used;
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == DUO_DT_BF16)
    duo::seq_merge_kernel<__nv_bfloat16><<<rows, 128, 0, s>>>(p);
  else
    duo::seq_merge_kernel<__half><<<rows, 128, 0, s>>>(p);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

}  // extern "C"
