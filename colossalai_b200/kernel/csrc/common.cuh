// Shared device helpers for the sm_90a kernel set (colossalai_b200).
// Replaces the reference's csrc/funcs/*_functor.h + common/{micros,vec_type_traits,mp_type_traits}.h with a
// much smaller surface: 16-byte vector I/O, fp32 math, warp/block reductions, and a runtime dtype switch.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>

#define CB_DEVICE __device__ __forceinline__
#define CB_HOST_DEVICE __host__ __device__ __forceinline__

// dtype codes shared with python (ops/_dtypes.py)
enum CbDtype : int { CB_F32 = 0, CB_F16 = 1, CB_BF16 = 2, CB_F8E4M3 = 3, CB_F8E5M2 = 4 };

#define CB_DISPATCH_FLOAT(code, T, ...)                                \
  switch (code) {                                                      \
    case CB_F32: { using T = float; __VA_ARGS__; break; }              \
    case CB_F16: { using T = __half; __VA_ARGS__; break; }             \
    case CB_BF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }     \
    default: return (int)cudaErrorInvalidValue;                        \
  }

#define CB_DISPATCH_HALF(code, T, ...)                                 \
  switch (code) {                                                      \
    case CB_F16: { using T = __half; __VA_ARGS__; break; }             \
    case CB_BF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }     \
    default: return (int)cudaErrorInvalidValue;                        \
  }

#define CB_LAUNCH_CHECK() (int)cudaGetLastError()

template <typename T> CB_DEVICE float to_f32(T v);
template <> CB_DEVICE float to_f32<float>(float v) { return v; }
template <> CB_DEVICE float to_f32<__half>(__half v) { return __half2float(v); }
template <> CB_DEVICE float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> CB_DEVICE T from_f32(float v);
template <> CB_DEVICE float from_f32<float>(float v) { return v; }
template <> CB_DEVICE __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> CB_DEVICE __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// two consecutive elements <-> two floats (8-byte fp32 / 4-byte 16-bit accesses; the address is 2-element aligned)
CB_DEVICE float2 to_f32x2(const float* p) { return *reinterpret_cast<const float2*>(p); }
CB_DEVICE float2 to_f32x2(const __nv_bfloat16* p) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p)); }
CB_DEVICE float2 to_f32x2(const __half* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }
CB_DEVICE void store_f32x2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
CB_DEVICE void store_f32x2(__nv_bfloat16* p, float a, float b) {
  *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(a, b);
}
CB_DEVICE void store_f32x2(__half* p, float a, float b) { *reinterpret_cast<__half2*>(p) = __floats2half2_rn(a, b); }

// A 16-byte vector of T (4 floats / 8 halves).
template <typename T> struct Vec16 {
  static constexpr int N = 16 / sizeof(T);
  union { uint4 raw; T v[N]; };
  CB_DEVICE void load(const T* p) { raw = *reinterpret_cast<const uint4*>(p); }
  CB_DEVICE void load_nc(const T* p) {
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(raw.x), "=r"(raw.y), "=r"(raw.z), "=r"(raw.w) : "l"(p));
  }
  CB_DEVICE void store(T* p) const { *reinterpret_cast<uint4*>(p) = raw; }
  CB_DEVICE void store_na(T* p) const {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(raw.x), "r"(raw.y), "r"(raw.z), "r"(raw.w) : "memory");
  }
  CB_DEVICE float get(int i) const { return to_f32<T>(v[i]); }
  CB_DEVICE void set(int i, float f) { v[i] = from_f32<T>(f); }
};

CB_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
CB_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum of up to two values; result broadcast to all threads.  `smem` needs 2*32 floats.
template <int NV> CB_DEVICE void block_sum(float (&vals)[NV], float* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) vals[i] = warp_sum(vals[i]);
  if (nwarps == 1) return;
  __syncthreads();  // protect smem reuse across calls
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) smem[i * 32 + warp] = vals[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float x = lane < nwarps ? smem[i * 32 + lane] : 0.f;
    vals[i] = warp_sum(x);
  }
}

CB_DEVICE float block_max(float v, float* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  if (nwarps == 1) return v;
  __syncthreads();
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  float x = lane < nwarps ? smem[lane] : -INFINITY;
  return warp_max(x);
}

static inline int cb_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;   // H100 SXM
  }
  return n;
}
