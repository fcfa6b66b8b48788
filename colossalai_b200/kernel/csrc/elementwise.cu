// Fused elementwise kernels for sm_90a: SwiGLU / GeGLU fwd+bwd on a packed [rows, 2*I] gate|up buffer,
// RoPE (half-rotation layout) applied in place to the q and k head ranges of a packed QKV buffer (fwd and bwd),
// bias+GELU fwd/bwd, bias+dropout+residual add, scale+inf/nan check.
//
// Capability parity: reference silu_and_mul (extensions/csrc/kernel/cuda/activation_kernel.cu, N16),
// rotary_embedding (fused_rotary_emb_and_cache_kernel.cu, N15), Triton LlamaActCombine
// (kernel/triton/llama_act_combine_kernel.py), TorchScript bias_gelu / bias_dropout_add (kernel/jit/*.py),
// multi_tensor_scale (N7).  All are pure HBM-bandwidth kernels: 16-byte vector I/O, grid-stride, fp32 math.
#include "common.cuh"

CB_DEVICE float silu_f(float x) { return x / (1.f + __expf(-x)); }
CB_DEVICE float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }
// tanh-approximated GELU, 0.5 x (1 + tanh u) with u = k (x + 0.044715 x^3), evaluated as x * sigmoid(2u).  The two
// are equal, but `tanhf` compiles to the tanh.approx unit under --use_fast_math (relative error 2^-11), and
// 1 + tanh u cancels for negative x; the sigmoid form has neither problem.
CB_DEVICE float gelu_tanh_f(float x) {
  const float k = 0.7978845608028654f;
  return x * sigmoid_f(2.f * k * (x + 0.044715f * x * x * x));
}
// d/dx = s + x * 2 s (1 - s) * u'  with s = sigmoid(2u)  (0.5 (1 + tanh u) = s, 1 - tanh^2 u = 4 s (1 - s))
CB_DEVICE float gelu_tanh_grad_f(float x) {
  const float k = 0.7978845608028654f;
  const float s = sigmoid_f(2.f * k * (x + 0.044715f * x * x * x));
  return s + 2.f * x * s * (1.f - s) * k * (1.f + 3.f * 0.044715f * x * x);
}
CB_DEVICE float gelu_erf_f(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }
CB_DEVICE float gelu_erf_grad_f(float x) {
  return 0.5f * (1.f + erff(x * 0.7071067811865476f)) + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}

// act: 0 = silu, 1 = gelu(tanh), 2 = gelu(erf)
template <int ACT> CB_DEVICE float act_f(float x) {
  return ACT == 0 ? silu_f(x) : (ACT == 1 ? gelu_tanh_f(x) : gelu_erf_f(x));
}
template <int ACT> CB_DEVICE float act_grad_f(float x) {
  if (ACT == 0) { const float s = sigmoid_f(x); return s * (1.f + x * (1.f - s)); }
  return ACT == 1 ? gelu_tanh_grad_f(x) : gelu_erf_grad_f(x);
}

template <typename T, int ACT>
__global__ void __launch_bounds__(256) glu_fwd_kernel(const T* __restrict__ gu, T* __restrict__ out, int64_t rows,
                                                      int I, const int64_t* __restrict__ row_limit) {
  constexpr int VEC = Vec16<T>::N;
  // row_limit (device scalar, optional): only the first *row_limit rows hold data - expert-parallel receive buffers are
  // sized for the worst case and the number of rows that actually arrived is only known on the device
  if (row_limit != nullptr) rows = min(rows, *row_limit);
  const int64_t vec_per_row = I / VEC, total = rows * vec_per_row;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / vec_per_row;
    const int c = (int)(idx - r * vec_per_row) * VEC;
    Vec16<T> g, u, o;
    g.load_nc(gu + r * 2 * I + c);
    u.load_nc(gu + r * 2 * I + I + c);
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.set(i, act_f<ACT>(g.get(i)) * u.get(i));
    o.store_na(out + r * I + c);
  }
}

template <typename T, int ACT>
__global__ void __launch_bounds__(256) glu_bwd_kernel(const T* __restrict__ dout, const T* __restrict__ gu,
                                                      T* __restrict__ dgu, int64_t rows, int I,
                                                      const int64_t* __restrict__ row_limit) {
  constexpr int VEC = Vec16<T>::N;
  if (row_limit != nullptr) rows = min(rows, *row_limit);
  const int64_t vec_per_row = I / VEC, total = rows * vec_per_row;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / vec_per_row;
    const int c = (int)(idx - r * vec_per_row) * VEC;
    Vec16<T> g, u, d, dg, du;
    g.load_nc(gu + r * 2 * I + c);
    u.load_nc(gu + r * 2 * I + I + c);
    d.load_nc(dout + r * I + c);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float gf = g.get(i), uf = u.get(i), df = d.get(i);
      dg.set(i, df * uf * act_grad_f<ACT>(gf));
      du.set(i, df * act_f<ACT>(gf));
    }
    dg.store_na(dgu + r * 2 * I + c);
    du.store_na(dgu + r * 2 * I + I + c);
  }
}

// RoPE in place on heads [0, n_rot_heads) of each token row of `qkv` ([T, row_stride] elements; head h starts at
// h*D).  cos/sin: fp32 caches [max_pos, D/2]; pos: int64 [T] (nullptr -> position = token index % seq_len_mod).
// sign = +1 forward, -1 backward (inverse rotation = transpose of the rotation matrix).
template <typename T>
__global__ void __launch_bounds__(256) rope_kernel(T* __restrict__ qkv, const int64_t* __restrict__ pos,
                                                   const float* __restrict__ cos_c, const float* __restrict__ sin_c,
                                                   int64_t T_tokens, int64_t row_stride, int n_rot_heads, int D,
                                                   int rot_dim, float sign, int interleaved) {
  constexpr int VEC = Vec16<T>::N;
  const int half = rot_dim / 2;
  const int vec_per_head = half / VEC;  // each work item rotates VEC (x1,x2) pairs
  const int64_t total = T_tokens * n_rot_heads * vec_per_head;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(idx % vec_per_head);
    const int64_t th = idx / vec_per_head;
    const int h = (int)(th % n_rot_heads);
    const int64_t t = th / n_rot_heads;
    const int64_t p = pos ? pos[t] : t;
    T* base = qkv + t * row_stride + (int64_t)h * D;
    const float* cp = cos_c + p * half + v * VEC;
    const float* sp = sin_c + p * half + v * VEC;
    if (!interleaved) {
      Vec16<T> x1, x2, o1, o2;
      x1.load(base + v * VEC);
      x2.load(base + half + v * VEC);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float c = cp[i], s = sp[i] * sign, a = x1.get(i), b = x2.get(i);
        o1.set(i, a * c - b * s);
        o2.set(i, b * c + a * s);
      }
      o1.store(base + v * VEC);
      o2.store(base + half + v * VEC);
    } else {
      // GPT-J / ChatGLM style: pairs are adjacent elements (2i, 2i+1); one item covers 2*VEC elements
      Vec16<T> a, b;
      a.load(base + 2 * v * VEC);
      b.load(base + 2 * v * VEC + VEC);
#pragma unroll
      for (int i = 0; i < VEC; i += 2) {
        {
          const int pi = i / 2;
          const float c = cp[pi], s = sp[pi] * sign, x = a.get(i), y = a.get(i + 1);
          a.set(i, x * c - y * s);
          a.set(i + 1, y * c + x * s);
        }
        {
          const int pi = VEC / 2 + i / 2;
          const float c = cp[pi], s = sp[pi] * sign, x = b.get(i), y = b.get(i + 1);
          b.set(i, x * c - y * s);
          b.set(i + 1, y * c + x * s);
        }
      }
      a.store(base + 2 * v * VEC);
      b.store(base + 2 * v * VEC + VEC);
    }
  }
}

template <typename T, int ACT>
__global__ void __launch_bounds__(256) bias_act_fwd_kernel(const T* __restrict__ x, const T* __restrict__ bias,
                                                           T* __restrict__ y, int64_t rows, int H) {
  constexpr int VEC = Vec16<T>::N;
  const int64_t vpr = H / VEC, total = rows * vpr;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % vpr) * VEC;
    Vec16<T> xv, bv, o;
    xv.load_nc(x + idx * VEC);
    if (bias) bv.load(bias + c);
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.set(i, act_f<ACT>(xv.get(i) + (bias ? bv.get(i) : 0.f)));
    o.store_na(y + idx * VEC);
  }
}

template <typename T, int ACT>
__global__ void __launch_bounds__(256) bias_act_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                           const T* __restrict__ bias, T* __restrict__ dx,
                                                           int64_t rows, int H) {
  constexpr int VEC = Vec16<T>::N;
  const int64_t vpr = H / VEC, total = rows * vpr;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % vpr) * VEC;
    Vec16<T> xv, bv, dv, o;
    xv.load_nc(x + idx * VEC);
    dv.load_nc(dy + idx * VEC);
    if (bias) bv.load(bias + c);
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.set(i, dv.get(i) * act_grad_f<ACT>(xv.get(i) + (bias ? bv.get(i) : 0.f)));
    o.store_na(dx + idx * VEC);
  }
}

// out = in * scale ; sets *flag = 1 if any element is inf/nan (loss-scale unscale + overflow check)
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) scale_check_kernel(const TI* __restrict__ in, TO* __restrict__ out,
                                                          int64_t n, float scale, int* __restrict__ flag) {
  bool bad = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = to_f32<TI>(in[i]);
    if (!isfinite(v)) bad = true;
    out[i] = from_f32<TO>(v * scale);
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) *flag = 1;
}

static inline int ew_grid(int64_t items, int block) {
  int64_t g = (items + block - 1) / block;
  const int64_t cap = (int64_t)cb_num_sms() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" {

int cb_glu_fwd_bounded(const void* gu, void* out, int64_t rows, int I, int act, int dtype, const int64_t* row_limit, cudaStream_t s) {
  if (rows == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    const int64_t items = rows * (I / Vec16<T>::N);
    const int g = ew_grid(items, 256);
    if (act == 0) glu_fwd_kernel<T, 0><<<g, 256, 0, s>>>((const T*)gu, (T*)out, rows, I, row_limit);
    else if (act == 1) glu_fwd_kernel<T, 1><<<g, 256, 0, s>>>((const T*)gu, (T*)out, rows, I, row_limit);
    else glu_fwd_kernel<T, 2><<<g, 256, 0, s>>>((const T*)gu, (T*)out, rows, I, row_limit);
  });
  return CB_LAUNCH_CHECK();
}

int cb_glu_bwd_bounded(const void* dout, const void* gu, void* dgu, int64_t rows, int I, int act, int dtype,
               const int64_t* row_limit, cudaStream_t s) {
  if (rows == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    const int64_t items = rows * (I / Vec16<T>::N);
    const int g = ew_grid(items, 256);
    if (act == 0) glu_bwd_kernel<T, 0><<<g, 256, 0, s>>>((const T*)dout, (const T*)gu, (T*)dgu, rows, I, row_limit);
    else if (act == 1) glu_bwd_kernel<T, 1><<<g, 256, 0, s>>>((const T*)dout, (const T*)gu, (T*)dgu, rows, I, row_limit);
    else glu_bwd_kernel<T, 2><<<g, 256, 0, s>>>((const T*)dout, (const T*)gu, (T*)dgu, rows, I, row_limit);
  });
  return CB_LAUNCH_CHECK();
}

int cb_glu_fwd(const void* gu, void* out, int64_t rows, int I, int act, int dtype, cudaStream_t s) {
  return cb_glu_fwd_bounded(gu, out, rows, I, act, dtype, nullptr, s);
}

int cb_glu_bwd(const void* dout, const void* gu, void* dgu, int64_t rows, int I, int act, int dtype, cudaStream_t s) {
  return cb_glu_bwd_bounded(dout, gu, dgu, rows, I, act, dtype, nullptr, s);
}

int cb_rope(void* qkv, const int64_t* pos, const float* cos_c, const float* sin_c, int64_t tokens,
            int64_t row_stride, int n_rot_heads, int D, int rot_dim, float sign, int interleaved, int dtype,
            cudaStream_t s) {
  if (tokens == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    const int64_t items = tokens * n_rot_heads * ((rot_dim / 2) / Vec16<T>::N);
    rope_kernel<T><<<ew_grid(items, 256), 256, 0, s>>>((T*)qkv, pos, cos_c, sin_c, tokens, row_stride, n_rot_heads, D,
                                                      rot_dim, sign, interleaved);
  });
  return CB_LAUNCH_CHECK();
}

int cb_bias_act_fwd(const void* x, const void* bias, void* y, int64_t rows, int H, int act, int dtype,
                    cudaStream_t s) {
  if (rows == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    const int g = ew_grid(rows * (H / Vec16<T>::N), 256);
    if (act == 0) bias_act_fwd_kernel<T, 0><<<g, 256, 0, s>>>((const T*)x, (const T*)bias, (T*)y, rows, H);
    else if (act == 1) bias_act_fwd_kernel<T, 1><<<g, 256, 0, s>>>((const T*)x, (const T*)bias, (T*)y, rows, H);
    else bias_act_fwd_kernel<T, 2><<<g, 256, 0, s>>>((const T*)x, (const T*)bias, (T*)y, rows, H);
  });
  return CB_LAUNCH_CHECK();
}

int cb_bias_act_bwd(const void* dy, const void* x, const void* bias, void* dx, int64_t rows, int H, int act,
                    int dtype, cudaStream_t s) {
  if (rows == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    const int g = ew_grid(rows * (H / Vec16<T>::N), 256);
    if (act == 0) bias_act_bwd_kernel<T, 0><<<g, 256, 0, s>>>((const T*)dy, (const T*)x, (const T*)bias, (T*)dx, rows, H);
    else if (act == 1) bias_act_bwd_kernel<T, 1><<<g, 256, 0, s>>>((const T*)dy, (const T*)x, (const T*)bias, (T*)dx, rows, H);
    else bias_act_bwd_kernel<T, 2><<<g, 256, 0, s>>>((const T*)dy, (const T*)x, (const T*)bias, (T*)dx, rows, H);
  });
  return CB_LAUNCH_CHECK();
}

// in dtype -> out dtype with scale; flag (int32 device) set to 1 on inf/nan
int cb_scale_check(const void* in, void* out, int64_t n, float scale, int* flag, int in_dtype, int out_dtype,
                   cudaStream_t s) {
  if (n == 0) return 0;
  const int g = ew_grid(n, 256);
#define SC(TI, TO) scale_check_kernel<TI, TO><<<g, 256, 0, s>>>((const TI*)in, (TO*)out, n, scale, flag)
  if (in_dtype == CB_F32 && out_dtype == CB_F32) SC(float, float);
  else if (in_dtype == CB_BF16 && out_dtype == CB_F32) SC(__nv_bfloat16, float);
  else if (in_dtype == CB_F16 && out_dtype == CB_F32) SC(__half, float);
  else if (in_dtype == CB_F32 && out_dtype == CB_BF16) SC(float, __nv_bfloat16);
  else if (in_dtype == CB_F32 && out_dtype == CB_F16) SC(float, __half);
  else if (in_dtype == CB_BF16 && out_dtype == CB_BF16) SC(__nv_bfloat16, __nv_bfloat16);
  else if (in_dtype == CB_F16 && out_dtype == CB_F16) SC(__half, __half);
  else return (int)cudaErrorInvalidValue;
#undef SC
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
