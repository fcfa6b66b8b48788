// Fused (vocab-parallel) cross-entropy building blocks for sm_90a.
// One CTA per token row; the [T, V_local] logits are streamed with 16-byte loads.  Forward reads the logits twice
// (row max, then sum-exp relative to the GLOBAL max that python all-reduces in between); backward reads once and
// writes the gradient once.  Replaces the eager torch composition in the reference's DistCrossEntropy
// (colossalai/shardformer/layer/loss.py:25-127) which materialises exp(logits) and a one-hot mask.
#include "common.cuh"

template <typename T>
__global__ void __launch_bounds__(512) ce_row_max_kernel(const T* __restrict__ x, float* __restrict__ out, int V, int Vv) {
  constexpr int VEC = Vec16<T>::N;
  __shared__ float red[32];
  const T* row = x + (size_t)blockIdx.x * V;
  float m = -INFINITY;
  for (int c = threadIdx.x * VEC; c < Vv; c += blockDim.x * VEC) {
    Vec16<T> v;
    v.load_nc(row + c);
#pragma unroll
    for (int i = 0; i < VEC; ++i) if (c + i < Vv) m = fmaxf(m, v.get(i));
  }
  m = block_max(m, red);
  if (threadIdx.x == 0) out[blockIdx.x] = m;
}

template <typename T>
__global__ void __launch_bounds__(512) ce_sumexp_target_kernel(const T* __restrict__ x,
                                                               const int64_t* __restrict__ target,
                                                               const float* __restrict__ gmax, float* __restrict__ out,
                                                               int Trows, int V, int Vv, int64_t vocab_start,
                                                               int64_t ignore_index) {
  constexpr int VEC = Vec16<T>::N;
  __shared__ float red[64];
  const int r = blockIdx.x;
  const T* row = x + (size_t)r * V;
  const float m = gmax[r];
  float s[1] = {0.f};
  for (int c = threadIdx.x * VEC; c < Vv; c += blockDim.x * VEC) {
    Vec16<T> v;
    v.load_nc(row + c);
#pragma unroll
    for (int i = 0; i < VEC; ++i) if (c + i < Vv) s[0] += __expf(v.get(i) - m);
  }
  block_sum<1>(s, red);
  if (threadIdx.x == 0) {
    out[r] = s[0];
    const int64_t t = target[r];
    const int64_t local = t - vocab_start;
    float tl = 0.f;
    if (t != ignore_index && local >= 0 && local < Vv) tl = to_f32<T>(row[local]);
    out[Trows + r] = tl;
  }
}

template <typename T>
__global__ void __launch_bounds__(512) ce_softmax_grad_kernel(const T* __restrict__ x,
                                                              const int64_t* __restrict__ target,
                                                              const float* __restrict__ gmax,
                                                              const float* __restrict__ sumexp,
                                                              const float* __restrict__ row_scale, T* __restrict__ g,
                                                              int V, int Vv, int64_t vocab_start,
                                                              int64_t ignore_index) {
  constexpr int VEC = Vec16<T>::N;
  const int r = blockIdx.x;
  const T* row = x + (size_t)r * V;
  T* grow = g + (size_t)r * V;
  const int64_t t = target[r];
  const bool ignored = (t == ignore_index);
  const float m = gmax[r], inv = ignored ? 0.f : row_scale[r] / sumexp[r];
  const float sc = ignored ? 0.f : row_scale[r];
  const int64_t local = t - vocab_start;
  for (int c = threadIdx.x * VEC; c < V; c += blockDim.x * VEC) {
    Vec16<T> v, o;
    v.load_nc(row + c);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      float p = (c + i < Vv) ? __expf(v.get(i) - m) * inv : 0.f;
      if ((int64_t)(c + i) == local) p -= sc;
      o.set(i, p);
    }
    o.store_na(grow + c);
  }
}

extern "C" {

int cb_ce_row_max(const void* x, float* out, int T_, int V, int Vv, int dtype, cudaStream_t s) {
  if (T_ == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, { ce_row_max_kernel<T><<<T_, 512, 0, s>>>((const T*)x, out, V, Vv); });
  return CB_LAUNCH_CHECK();
}

int cb_ce_sumexp_target(const void* x, const int64_t* target, const float* gmax, float* out, int T_, int V, int Vv,
                        int64_t vocab_start, int64_t ignore_index, int dtype, cudaStream_t s) {
  if (T_ == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    ce_sumexp_target_kernel<T><<<T_, 512, 0, s>>>((const T*)x, target, gmax, out, T_, V, Vv, vocab_start, ignore_index);
  });
  return CB_LAUNCH_CHECK();
}

int cb_ce_softmax_grad(const void* x, const int64_t* target, const float* gmax, const float* sumexp,
                       const float* row_scale, void* g, int T_, int V, int Vv, int64_t vocab_start,
                       int64_t ignore_index, int dtype, cudaStream_t s) {
  if (T_ == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    ce_softmax_grad_kernel<T><<<T_, 512, 0, s>>>((const T*)x, target, gmax, sumexp, row_scale, (T*)g, V, Vv,
                                                vocab_start, ignore_index);
  });
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
