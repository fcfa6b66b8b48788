// Scaled masked softmax and scaled upper-triangular (causal) masked softmax, forward + backward.
// Behavioural parity: reference extensions/csrc/kernel/cuda/scaled_masked_softmax_kernel.cu (fwd :35, bwd :158) and
// scaled_upper_triang_masked_softmax_kernel.cu (fwd :35, bwd :157): y = softmax(scale * x masked_fill(mask, -10000)).
// Design here: one warp per row for sk <= 1024 (row lives in registers, two shuffles reductions), one CTA per row
// beyond that (no 2048-key limit as in the reference); fp32 math, 16-bit or fp32 I/O.
#include "common.cuh"

namespace {

constexpr float MASK_FILL = -10000.0f;

// ---- warp-per-row kernels (sk <= 32 * PER)
template <typename T, int PER, bool CAUSAL>
__global__ void __launch_bounds__(128) softmax_fwd_warp(const T* __restrict__ x, const uint8_t* __restrict__ mask,
                                                        T* __restrict__ y, float scale, int64_t rows, int sq, int sk,
                                                        int heads, int mask_batch_stride_is_one) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int q = (int)(row % sq);
  // mask [b, 1, sq, sk] (broadcast over heads); row index = ((b*heads + h)*sq + q)
  const int64_t b = row / ((int64_t)heads * sq);
  const uint8_t* mrow = mask ? mask + ((mask_batch_stride_is_one ? 0 : b) * sq + q) * (int64_t)sk : nullptr;
  const T* xr = x + row * sk;
  float v[PER];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int c = lane + i * 32;
    if (c < sk) {
      float t = to_f32<T>(xr[c]) * scale;
      if (CAUSAL) { if (c > q + (sk - sq)) t = -INFINITY; }
      else if (mrow && mrow[c]) t = MASK_FILL;
      v[i] = t;
    } else v[i] = -INFINITY;
    mx = fmaxf(mx, v[i]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    v[i] = (v[i] == -INFINITY) ? 0.f : __expf(v[i] - mx);
    sum += v[i];
  }
  sum = warp_sum(sum);
  const float inv = sum > 0.f ? 1.f / sum : 0.f;
  T* yr = y + row * sk;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int c = lane + i * 32;
    if (c < sk) yr[c] = from_f32<T>(v[i] * inv);
  }
}

// dx = scale * y * (dy - sum(dy * y))
template <typename T, int PER>
__global__ void __launch_bounds__(128) softmax_bwd_warp(const T* __restrict__ dy, const T* __restrict__ y, T* __restrict__ dx,
                                                        float scale, int64_t rows, int sk) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float g[PER], p[PER];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int c = lane + i * 32;
    g[i] = c < sk ? to_f32<T>(dy[row * sk + c]) : 0.f;
    p[i] = c < sk ? to_f32<T>(y[row * sk + c]) : 0.f;
    dot += g[i] * p[i];
  }
  dot = warp_sum(dot);
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int c = lane + i * 32;
    if (c < sk) dx[row * sk + c] = from_f32<T>(scale * p[i] * (g[i] - dot));
  }
}

// ---- CTA-per-row kernels (any sk)
template <typename T, bool CAUSAL>
__global__ void __launch_bounds__(256) softmax_fwd_block(const T* __restrict__ x, const uint8_t* __restrict__ mask,
                                                         T* __restrict__ y, float scale, int sq, int sk, int heads,
                                                         int mask_batch_stride_is_one) {
  const int64_t row = blockIdx.x;
  const int q = (int)(row % sq);
  const int64_t b = row / ((int64_t)heads * sq);
  const uint8_t* mrow = mask ? mask + ((mask_batch_stride_is_one ? 0 : b) * sq + q) * (int64_t)sk : nullptr;
  const T* xr = x + row * sk;
  T* yr = y + row * sk;
  __shared__ float red[64];
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < sk; c += blockDim.x) {
    float t = to_f32<T>(xr[c]) * scale;
    if (CAUSAL) { if (c > q + (sk - sq)) t = -INFINITY; }
    else if (mrow && mrow[c]) t = MASK_FILL;
    mx = fmaxf(mx, t);
  }
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = -INFINITY;
  for (int w = 0; w < (blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float s[1] = {0.f};
  for (int c = threadIdx.x; c < sk; c += blockDim.x) {
    float t = to_f32<T>(xr[c]) * scale;
    if (CAUSAL) { if (c > q + (sk - sq)) t = -INFINITY; }
    else if (mrow && mrow[c]) t = MASK_FILL;
    s[0] += (t == -INFINITY) ? 0.f : __expf(t - mx);
  }
  block_sum<1>(s, red);
  const float inv = s[0] > 0.f ? 1.f / s[0] : 0.f;
  for (int c = threadIdx.x; c < sk; c += blockDim.x) {
    float t = to_f32<T>(xr[c]) * scale;
    if (CAUSAL) { if (c > q + (sk - sq)) t = -INFINITY; }
    else if (mrow && mrow[c]) t = MASK_FILL;
    yr[c] = from_f32<T>((t == -INFINITY) ? 0.f : __expf(t - mx) * inv);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) softmax_bwd_block(const T* __restrict__ dy, const T* __restrict__ y, T* __restrict__ dx,
                                                         float scale, int sk) {
  const int64_t row = blockIdx.x;
  __shared__ float red[64];
  float d[1] = {0.f};
  for (int c = threadIdx.x; c < sk; c += blockDim.x) d[0] += to_f32<T>(dy[row * sk + c]) * to_f32<T>(y[row * sk + c]);
  block_sum<1>(d, red);
  for (int c = threadIdx.x; c < sk; c += blockDim.x) {
    const float p = to_f32<T>(y[row * sk + c]);
    dx[row * sk + c] = from_f32<T>(scale * p * (to_f32<T>(dy[row * sk + c]) - d[0]));
  }
}

template <typename T, bool CAUSAL>
int launch_fwd(const T* x, const uint8_t* mask, T* y, float scale, int64_t rows, int sq, int sk, int heads, int mb1,
               cudaStream_t st) {
  const int wpb = 4;
  const int grid = (int)((rows + wpb - 1) / wpb);
#define W(PER) softmax_fwd_warp<T, PER, CAUSAL><<<grid, wpb * 32, 0, st>>>(x, mask, y, scale, rows, sq, sk, heads, mb1)
  if (sk <= 32) W(1);
  else if (sk <= 64) W(2);
  else if (sk <= 128) W(4);
  else if (sk <= 256) W(8);
  else if (sk <= 512) W(16);
  else if (sk <= 1024) W(32);
  else softmax_fwd_block<T, CAUSAL><<<(unsigned)rows, 256, 0, st>>>(x, mask, y, scale, sq, sk, heads, mb1);
#undef W
  return CB_LAUNCH_CHECK();
}

template <typename T>
int launch_bwd(const T* dy, const T* y, T* dx, float scale, int64_t rows, int sk, cudaStream_t st) {
  const int wpb = 4;
  const int grid = (int)((rows + wpb - 1) / wpb);
#define W(PER) softmax_bwd_warp<T, PER><<<grid, wpb * 32, 0, st>>>(dy, y, dx, scale, rows, sk)
  if (sk <= 32) W(1);
  else if (sk <= 64) W(2);
  else if (sk <= 128) W(4);
  else if (sk <= 256) W(8);
  else if (sk <= 512) W(16);
  else if (sk <= 1024) W(32);
  else softmax_bwd_block<T><<<(unsigned)rows, 256, 0, st>>>(dy, y, dx, scale, sk);
#undef W
  return CB_LAUNCH_CHECK();
}

}  // namespace

extern "C" {

// x, y: [b, heads, sq, sk]; mask: uint8 [b or 1, 1, sq, sk] (nonzero = masked) or null
int cb_scaled_masked_softmax_fwd(const void* x, const void* mask, void* y, float scale, int b, int heads, int sq, int sk,
                                 int mask_b, int dtype, cudaStream_t st) {
  const int64_t rows = (int64_t)b * heads * sq;
  if (rows == 0 || sk == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    return launch_fwd<T, false>((const T*)x, (const uint8_t*)mask, (T*)y, scale, rows, sq, sk, heads, mask_b == 1, st);
  });
  return 0;
}

// x, y: [attn_batches, sq, sk] causal (key c visible to query q iff c <= q + sk - sq)
int cb_scaled_causal_softmax_fwd(const void* x, void* y, float scale, int attn_batches, int sq, int sk, int dtype,
                                 cudaStream_t st) {
  const int64_t rows = (int64_t)attn_batches * sq;
  if (rows == 0 || sk == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    return launch_fwd<T, true>((const T*)x, nullptr, (T*)y, scale, rows, sq, sk, 1, 1, st);
  });
  return 0;
}

int cb_scaled_softmax_bwd(const void* dy, const void* y, void* dx, float scale, int64_t rows, int sk, int dtype,
                          cudaStream_t st) {
  if (rows == 0 || sk == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, { return launch_bwd<T>((const T*)dy, (const T*)y, (T*)dx, scale, rows, sk, st); });
  return 0;
}

}  // extern "C"
