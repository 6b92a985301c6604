// Caller-side glue of the hot path (SURVEY.md §8f3): the residual add + RMSNorm pair and the SiLU*up product
// that sit between the attention / MLP GEMMs of every decoder layer.  In the reference these are ~20 tiny
// PyTorch kernels per layer (HF LlamaRMSNorm in fp32, flashinfer rmsnorm in the static path:
// duo_attn/patch/flashinfer_utils.py:9-26); at decode they are pure launch latency, at prefill pure HBM traffic.
// One launch each here, HF arithmetic preserved: norm in fp32, rounded to the activation dtype, THEN multiplied
// by the weight in that dtype; silu evaluated in fp32 and rounded before the product.
#include "duo_common.cuh"

namespace duo {

template <typename T>
struct EwCvt;
template <>
struct EwCvt<__nv_bfloat16> {
  __device__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <>
struct EwCvt<__half> {
  __device__ static float to_f(__half v) { return __half2float(v); }
  __device__ static __half from_f(float v) { return __float2half_rn(v); }
};

template <typename T>
struct alignas(16) Vec8 {
  T v[8];
};

// one CTA per row; hidden % 8 == 0
template <typename T>
__global__ void __launch_bounds__(256) add_rmsnorm_kernel(const T* __restrict__ x, const T* __restrict__ residual,
                                                          const T* __restrict__ weight, T* __restrict__ out_norm,
                                                          T* __restrict__ out_res, int hidden, float eps) {
  extern __shared__ float s_row[];  // hidden floats (the summed row, already rounded to T)
  __shared__ float s_part[8];
  const long long row = blockIdx.x;
  const T* xr = x + row * hidden;
  const T* rr = residual ? residual + row * hidden : nullptr;
  float ss = 0.f;
  for (int i = threadIdx.x * 8; i < hidden; i += blockDim.x * 8) {
    Vec8<T> a = *reinterpret_cast<const Vec8<T>*>(xr + i);
    if (rr) {
      const Vec8<T> b = *reinterpret_cast<const Vec8<T>*>(rr + i);
#pragma unroll
      for (int k = 0; k < 8; ++k) a.v[k] = EwCvt<T>::from_f(EwCvt<T>::to_f(b.v[k]) + EwCvt<T>::to_f(a.v[k]));
      if (out_res) *reinterpret_cast<Vec8<T>*>(out_res + row * hidden + i) = a;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float f = EwCvt<T>::to_f(a.v[k]);
      s_row[i + k] = f;
      ss += f * f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += (w < (int)(blockDim.x >> 5)) ? s_part[w] : 0.f;
  const float inv = rsqrtf(tot / (float)hidden + eps);
  for (int i = threadIdx.x * 8; i < hidden; i += blockDim.x * 8) {
    const Vec8<T> w = *reinterpret_cast<const Vec8<T>*>(weight + i);
    Vec8<T> o;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const T n = EwCvt<T>::from_f(s_row[i + k] * inv);
      o.v[k] = EwCvt<T>::from_f(EwCvt<T>::to_f(w.v[k]) * EwCvt<T>::to_f(n));
    }
    *reinterpret_cast<Vec8<T>*>(out_norm + row * hidden + i) = o;
  }
}

// gate_up: [rows][2*inter] (gate | up), out: [rows][inter]
template <typename T>
__global__ void __launch_bounds__(256) silu_mul_kernel(const T* __restrict__ gate_up, T* __restrict__ out, long long rows,
                                                       int inter) {
  const long long per_row = inter / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * per_row) return;
  const long long row = idx / per_row;
  const int c = (int)(idx % per_row) * 8;
  const Vec8<T> g = *reinterpret_cast<const Vec8<T>*>(gate_up + row * 2 * inter + c);
  const Vec8<T> u = *reinterpret_cast<const Vec8<T>*>(gate_up + row * 2 * inter + inter + c);
  Vec8<T> o;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float gf = EwCvt<T>::to_f(g.v[k]);
    const T act = EwCvt<T>::from_f(gf / (1.0f + __expf(-gf)));
    o.v[k] = EwCvt<T>::from_f(EwCvt<T>::to_f(act) * EwCvt<T>::to_f(u.v[k]));
  }
  *reinterpret_cast<Vec8<T>*>(out + row * inter + c) = o;
}

int launch_add_rmsnorm(const void* x, const void* residual, const void* weight, void* out_norm, void* out_res,
                       long long rows, int hidden, float eps, int dtype, cudaStream_t stream) {
  if (rows == 0) return DUO_OK;
  const size_t smem = (size_t)hidden * sizeof(float);
  // the 48 KB default limit covers dynamic + static shared memory (s_part): hidden >= 12288 needs the opt-in (the API
  // accepts up to 16384 = 64 KB)
  if (smem + kStaticSmemHeadroom > 48 * 1024) {
    static unsigned long long mask_bf = 0, mask_h = 0;
    const int rc = dtype == DUO_DT_BF16 ? ensure_dyn_smem(add_rmsnorm_kernel<__nv_bfloat16>, 64 * 1024, &mask_bf)
                                        : ensure_dyn_smem(add_rmsnorm_kernel<__half>, 64 * 1024, &mask_h);
    if (rc) return rc;
  }
  if (dtype == DUO_DT_BF16) {
    add_rmsnorm_kernel<__nv_bfloat16><<<(unsigned)rows, 256, smem, stream>>>(
        (const __nv_bfloat16*)x, (const __nv_bfloat16*)residual, (const __nv_bfloat16*)weight, (__nv_bfloat16*)out_norm,
        (__nv_bfloat16*)out_res, hidden, eps);
  } else {
    add_rmsnorm_kernel<__half><<<(unsigned)rows, 256, smem, stream>>>((const __half*)x, (const __half*)residual,
                                                                      (const __half*)weight, (__half*)out_norm,
                                                                      (__half*)out_res, hidden, eps);
  }
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

int launch_silu_mul(const void* gate_up, void* out, long long rows, int inter, int dtype, cudaStream_t stream) {
  if (rows == 0) return DUO_OK;
  const long long n = rows * (inter / 8);
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (dtype == DUO_DT_BF16)
    silu_mul_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>((const __nv_bfloat16*)gate_up, (__nv_bfloat16*)out, rows, inter);
  else
    silu_mul_kernel<__half><<<blocks, 256, 0, stream>>>((const __half*)gate_up, (__half*)out, rows, inter);
  DUO_CUDA_TRY(cudaGetLastError());
  return DUO_OK;
}

}  // namespace duo
