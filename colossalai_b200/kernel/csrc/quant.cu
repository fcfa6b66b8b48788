// FP8 scaled quantisation kernels (per-tensor and per-row scaling) for fp8 communication / fp8 linear.
// Reference behaviour: colossalai/quantization/fp8.py:51-118 (cast_to_fp8 / cast_from_fp8: scale = fp8_max / amax,
// scale_inv returned to the caller).  Here the amax reduction and the cast are native kernels; the per-row variant is a
// single pass (row kept in registers between the reduction and the cast).
#include "common.cuh"

namespace {

template <int FMT> CB_DEVICE uint8_t f32_to_fp8(float v) {
  return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, FMT == 0 ? __NV_E4M3 : __NV_E5M2);
}
template <int FMT> CB_DEVICE float fp8_to_f32(uint8_t b) {
  __half_raw h = __nv_cvt_fp8_to_halfraw(b, FMT == 0 ? __NV_E4M3 : __NV_E5M2);
  return __half2float(*reinterpret_cast<__half*>(&h));
}

// ---- per-tensor amax: grid-stride, one atomicMax on the float bit pattern (values are >= 0)
template <typename T>
__global__ void __launch_bounds__(512) absmax_kernel(const T* __restrict__ x, int64_t n, float* __restrict__ amax) {
  constexpr int V = Vec16<T>::N;
  float m = 0.f;
  const int64_t nvec = n / V;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    Vec16<T> v; v.load_nc(x + i * V);
#pragma unroll
    for (int j = 0; j < V; ++j) m = fmaxf(m, fabsf(v.get(j)));
  }
  for (int64_t i = nvec * V + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(to_f32<T>(x[i])));
  m = warp_max(m);
  __shared__ float sm[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sm[warp] = m;
  __syncthreads();
  if (warp == 0) {
    m = lane < (blockDim.x >> 5) ? sm[lane] : 0.f;
    m = warp_max(m);
    if (lane == 0) atomicMax(reinterpret_cast<unsigned int*>(amax), __float_as_uint(m));
  }
}

// ---- per-tensor cast: scale = fp8_max / max(amax, tiny); writes scale_inv[0] from block 0
template <typename T, int FMT>
__global__ void __launch_bounds__(512) cast_to_fp8_kernel(const T* __restrict__ x, uint8_t* __restrict__ out, int64_t n,
                                                          const float* __restrict__ amax, float* __restrict__ scale_inv,
                                                          float fp8_max) {
  constexpr int V = Vec16<T>::N;
  float a = *amax;
  a = a > 0.f ? a : 1.f;
  const float scale = fp8_max / a;
  if (blockIdx.x == 0 && threadIdx.x == 0) *scale_inv = a / fp8_max;
  const int64_t nvec = n / V;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    Vec16<T> v; v.load_nc(x + i * V);
    uint8_t o[V];
#pragma unroll
    for (int j = 0; j < V; ++j) o[j] = f32_to_fp8<FMT>(v.get(j) * scale);
    if (V == 8) *reinterpret_cast<uint2*>(out + i * V) = *reinterpret_cast<uint2*>(o);
    else *reinterpret_cast<uint32_t*>(out + i * V) = *reinterpret_cast<uint32_t*>(o);
  }
  for (int64_t i = nvec * V + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = f32_to_fp8<FMT>(to_f32<T>(x[i]) * scale);
}

// ---- per-row (per-channel) single pass: one CTA per row
template <typename T, int FMT>
__global__ void __launch_bounds__(256) cast_to_fp8_rows_kernel(const T* __restrict__ x, uint8_t* __restrict__ out,
                                                               int cols, int64_t ld, float* __restrict__ scale_inv,
                                                               float fp8_max) {
  const T* row = x + (int64_t)blockIdx.x * ld;
  uint8_t* orow = out + (int64_t)blockIdx.x * cols;
  float m = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, fabsf(to_f32<T>(row[c])));
  m = warp_max(m);
  __shared__ float sm[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sm[warp] = m;
  __syncthreads();
  m = 0.f;
  for (int w = 0; w < (blockDim.x >> 5); ++w) m = fmaxf(m, sm[w]);
  m = m > 0.f ? m : 1.f;
  const float scale = fp8_max / m;
  if (threadIdx.x == 0) scale_inv[blockIdx.x] = m / fp8_max;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) orow[c] = f32_to_fp8<FMT>(to_f32<T>(row[c]) * scale);
}

template <typename T, int FMT>
__global__ void __launch_bounds__(512) cast_from_fp8_kernel(const uint8_t* __restrict__ x, T* __restrict__ out, int64_t n,
                                                            const float* __restrict__ scale_inv, int cols) {
  // cols > 0: per-row scales (scale_inv[row]); cols == 0: per-tensor
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 4; i < n; i += (int64_t)gridDim.x * blockDim.x * 4) {
    if (i + 4 <= n && (cols == 0 || cols % 4 == 0)) {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(x + i);
      const float s = cols ? scale_inv[i / cols] : *scale_inv;
#pragma unroll
      for (int j = 0; j < 4; ++j) out[i + j] = from_f32<T>(fp8_to_f32<FMT>((w >> (8 * j)) & 0xff) * s);
    } else {
      for (int64_t k = i; k < n && k < i + 4; ++k)
        out[k] = from_f32<T>(fp8_to_f32<FMT>(x[k]) * (cols ? scale_inv[k / cols] : *scale_inv));
    }
  }
}

inline int grid_for(int64_t n, int per_block) {
  int64_t g = (n + per_block - 1) / per_block;
  return (int)(g < 1 ? 1 : (g > cb_num_sms() * 8 ? cb_num_sms() * 8 : g));
}

}  // namespace

extern "C" {

// amax must be zero-initialised by the caller (cudaMemsetAsync is issued here for convenience).
int cb_fp8_quant_tensor(const void* x, void* out, int64_t n, float* amax, float* scale_inv, int dtype, int fmt,
                        cudaStream_t s) {
  if (n == 0) return 0;
  cudaMemsetAsync(amax, 0, sizeof(float), s);
  const float fp8_max = fmt == 0 ? 448.f : 57344.f;
  CB_DISPATCH_FLOAT(dtype, T, {
    absmax_kernel<T><<<grid_for(n, 512 * Vec16<T>::N), 512, 0, s>>>((const T*)x, n, amax);
    if (fmt == 0)
      cast_to_fp8_kernel<T, 0><<<grid_for(n, 512 * Vec16<T>::N), 512, 0, s>>>((const T*)x, (uint8_t*)out, n, amax,
                                                                            scale_inv, fp8_max);
    else
      cast_to_fp8_kernel<T, 1><<<grid_for(n, 512 * Vec16<T>::N), 512, 0, s>>>((const T*)x, (uint8_t*)out, n, amax,
                                                                            scale_inv, fp8_max);
  });
  return CB_LAUNCH_CHECK();
}

int cb_fp8_quant_rows(const void* x, void* out, int rows, int cols, int64_t ld, float* scale_inv, int dtype, int fmt,
                      cudaStream_t s) {
  if (rows == 0 || cols == 0) return 0;
  const float fp8_max = fmt == 0 ? 448.f : 57344.f;
  CB_DISPATCH_FLOAT(dtype, T, {
    if (fmt == 0)
      cast_to_fp8_rows_kernel<T, 0><<<rows, 256, 0, s>>>((const T*)x, (uint8_t*)out, cols, ld, scale_inv, fp8_max);
    else
      cast_to_fp8_rows_kernel<T, 1><<<rows, 256, 0, s>>>((const T*)x, (uint8_t*)out, cols, ld, scale_inv, fp8_max);
  });
  return CB_LAUNCH_CHECK();
}

// cols == 0 -> per-tensor scale_inv[0]; else per-row scale_inv[i / cols]
int cb_fp8_dequant(const void* x, void* out, int64_t n, const float* scale_inv, int cols, int dtype, int fmt,
                   cudaStream_t s) {
  if (n == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    if (fmt == 0)
      cast_from_fp8_kernel<T, 0><<<grid_for(n, 2048), 512, 0, s>>>((const uint8_t*)x, (T*)out, n, scale_inv, cols);
    else
      cast_from_fp8_kernel<T, 1><<<grid_for(n, 2048), 512, 0, s>>>((const uint8_t*)x, (T*)out, n, scale_inv, cols);
  });
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
