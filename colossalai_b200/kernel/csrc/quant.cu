// FP8 scaled quantisation kernels (per-tensor and per-row scaling) for fp8 communication / fp8 linear, and the int8
// per-token (or static-scale) activation quantiser of the SmoothQuant W8A8 linear.
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

constexpr int FMT_INT8 = 2;

CB_DEVICE uint8_t to_int8(float v, float s) {
  return (uint8_t)(int8_t)fminf(fmaxf(rintf(__fdiv_rn(v, s)), -127.f), 127.f);
}

// int8 rows: 16-byte loads when the row allows them (the scalar loop leaves a long decode row latency-bound)
template <typename T> CB_DEVICE bool vec_row(const T* row, int cols) {
  return cols % Vec16<T>::N == 0 && reinterpret_cast<uintptr_t>(row) % 16 == 0;
}
template <typename T> CB_DEVICE float int8_row_absmax(const T* row, int cols) {
  constexpr int V = Vec16<T>::N;
  float m = 0.f;
  if (vec_row(row, cols)) {
    for (int c = threadIdx.x * V; c < cols; c += blockDim.x * V) {
      Vec16<T> v; v.load(row + c);
#pragma unroll
      for (int j = 0; j < V; ++j) m = fmaxf(m, fabsf(v.get(j)));
    }
  } else {
    for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, fabsf(to_f32<T>(row[c])));
  }
  return m;
}
template <typename T> CB_DEVICE void int8_row_store(const T* row, uint8_t* orow, int cols, float s) {
  constexpr int V = Vec16<T>::N;
  if (vec_row(row, cols)) {
    for (int c = threadIdx.x * V; c < cols; c += blockDim.x * V) {
      Vec16<T> v; v.load(row + c);
      uint8_t o[V];
#pragma unroll
      for (int j = 0; j < V; ++j) o[j] = to_int8(v.get(j), s);
      if (V == 8) *reinterpret_cast<uint2*>(orow + c) = *reinterpret_cast<uint2*>(o);
      else *reinterpret_cast<uint32_t*>(orow + c) = *reinterpret_cast<uint32_t*>(o);
    }
  } else {
    for (int c = threadIdx.x; c < cols; c += blockDim.x) orow[c] = to_int8(to_f32<T>(row[c]), s);
  }
}

// ---- per-row (per-channel) single pass: one CTA per row.  FMT 0 / 1: fp8 E4M3 / E5M2 with scale_inv = amax / fp8_max.
// FMT_INT8: q = clamp(rint(x / s), -127, 127) with s = max(amax, 1e-8) * fl(1 / 127) written to scale_inv (the rounding
// steps of the PyTorch per-token quantiser on the GPU, which multiplies by the reciprocal of a host scalar divisor), or,
// with static_scale, s = *static_scale and no reduction (scale_inv is not written).
template <typename T, int FMT>
__global__ void __launch_bounds__(256) cast_to_fp8_rows_kernel(const T* __restrict__ x, uint8_t* __restrict__ out,
                                                               int cols, int64_t ld, float* __restrict__ scale_inv,
                                                               float fp8_max, const float* __restrict__ static_scale) {
  const T* row = x + (int64_t)blockIdx.x * ld;
  uint8_t* orow = out + (int64_t)blockIdx.x * cols;
  if (FMT == FMT_INT8 && static_scale) {
    int8_row_store(row, orow, cols, __ldg(static_scale));
    return;
  }
  float m = 0.f;
  if constexpr (FMT == FMT_INT8)
    m = int8_row_absmax(row, cols);
  else
    for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, fabsf(to_f32<T>(row[c])));
  m = warp_max(m);
  __shared__ float sm[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sm[warp] = m;
  __syncthreads();
  m = 0.f;
  for (int w = 0; w < (blockDim.x >> 5); ++w) m = fmaxf(m, sm[w]);
  if constexpr (FMT == FMT_INT8) {
    const float s = __fmul_rn(fmaxf(m, 1e-8f), 0x1.020408p-7f);   // fl(1 / 127), not left to fast-math division
    if (threadIdx.x == 0) scale_inv[blockIdx.x] = s;
    int8_row_store(row, orow, cols, s);
  } else {
    m = m > 0.f ? m : 1.f;
    const float scale = fp8_max / m;
    if (threadIdx.x == 0) scale_inv[blockIdx.x] = m / fp8_max;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) orow[c] = f32_to_fp8<FMT>(to_f32<T>(row[c]) * scale);
  }
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
      cast_to_fp8_rows_kernel<T, 0><<<rows, 256, 0, s>>>((const T*)x, (uint8_t*)out, cols, ld, scale_inv, fp8_max,
                                                         nullptr);
    else
      cast_to_fp8_rows_kernel<T, 1><<<rows, 256, 0, s>>>((const T*)x, (uint8_t*)out, cols, ld, scale_inv, fp8_max,
                                                         nullptr);
  });
  return CB_LAUNCH_CHECK();
}

// W8A8 activations: x [rows, cols] (row stride ld elements, fp32 / fp16 / bf16) -> int8 out [rows, cols] (contiguous).
// static_scale null: per-row scales to scale[rows] (fp32); else the device fp32 scalar divides every row.
int cb_int8_quant_rows(const void* x, void* out, int rows, int cols, int64_t ld, float* scale,
                       const float* static_scale, int dtype, cudaStream_t s) {
  if (rows < 0 || cols < 0 || ld < cols || (!scale && !static_scale)) return (int)cudaErrorInvalidValue;
  if (rows == 0 || cols == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    cast_to_fp8_rows_kernel<T, FMT_INT8><<<rows, 256, 0, s>>>((const T*)x, (uint8_t*)out, cols, ld, scale, 0.f,
                                                              static_scale);
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
