// Fused RMSNorm / LayerNorm forward + backward for sm_90a (memory-bound: 16-byte vector I/O, row in registers,
// fp32 statistics, one pass over HBM per tensor).
//
// Capability parity: reference apex FusedRMSNorm/FusedLayerNorm usage (shardformer/layer/normalization.py:27-135),
// extensions/csrc/kernel/cuda/layer_norm_kernel.cu (N8) and rms_layernorm_kernel.cu (N17: residual-add fusion).
// Design here is new: a single kernel handles (optional) residual-add + norm and emits rstd for backward;
// backward is a persistent grid that keeps dgamma/dbeta partials in registers and a tiny second pass reduces them.
#include "common.cuh"

constexpr int MAX_ITERS_LIMIT = 4;

template <typename T, bool HAS_RES, int MAX_ITERS>
__global__ void __launch_bounds__(1024) rmsnorm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ res_in,
                                                           const T* __restrict__ w, T* __restrict__ y,
                                                           T* __restrict__ res_out, float* __restrict__ rstd_out,
                                                           int rows, int H, float eps) {
  constexpr int VEC = Vec16<T>::N;
  __shared__ float red[64];
  const int row = blockIdx.x;
  if (row >= rows) return;
  const size_t base = (size_t)row * H;
  Vec16<T> hv[MAX_ITERS];
  float ss[1] = {0.f};
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) {
      hv[it].load_nc(x + base + col);
      if (HAS_RES) {
        Vec16<T> r;
        r.load_nc(res_in + base + col);
#pragma unroll
        for (int i = 0; i < VEC; ++i) hv[it].set(i, hv[it].get(i) + r.get(i));
        hv[it].store(res_out + base + col);
      }
#pragma unroll
      for (int i = 0; i < VEC; ++i) { float f = hv[it].get(i); ss[0] += f * f; }
    }
  }
  block_sum<1>(ss, red);
  const float rstd = rsqrtf(ss[0] / (float)H + eps);
  if (threadIdx.x == 0 && rstd_out) rstd_out[row] = rstd;
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) {
      Vec16<T> wv, o;
      wv.load(w + col);
#pragma unroll
      for (int i = 0; i < VEC; ++i) o.set(i, hv[it].get(i) * rstd * wv.get(i));
      o.store_na(y + base + col);
    }
  }
}

// dx = rstd * (w*dy - xhat * mean(w*dy*xhat)) (+ dres);   dw_partial[cta] = sum_rows dy * xhat
template <typename T, bool HAS_DRES, int MAX_ITERS>
__global__ void __launch_bounds__(1024) rmsnorm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ h,
                                                           const T* __restrict__ w, const float* __restrict__ rstd,
                                                           const T* __restrict__ dres, T* __restrict__ dx,
                                                           float* __restrict__ dw_partial, int rows, int H) {
  constexpr int VEC = Vec16<T>::N;
  __shared__ float red[64];
  float dw_acc[MAX_ITERS][VEC];
  Vec16<T> wv[MAX_ITERS];
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) wv[it].load(w + col);
#pragma unroll
    for (int i = 0; i < VEC; ++i) dw_acc[it][i] = 0.f;
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const size_t base = (size_t)row * H;
    const float rs = rstd[row];
    Vec16<T> dyv[MAX_ITERS], hv[MAX_ITERS];
    float c[1] = {0.f};
#pragma unroll
    for (int it = 0; it < MAX_ITERS; ++it) {
      const int col = (it * blockDim.x + threadIdx.x) * VEC;
      if (col < H) {
        dyv[it].load_nc(dy + base + col);
        hv[it].load_nc(h + base + col);
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float xhat = hv[it].get(i) * rs, g = dyv[it].get(i);
          c[0] += g * wv[it].get(i) * xhat;
          dw_acc[it][i] += g * xhat;
        }
      }
    }
    block_sum<1>(c, red);
    const float c1 = c[0] / (float)H;
#pragma unroll
    for (int it = 0; it < MAX_ITERS; ++it) {
      const int col = (it * blockDim.x + threadIdx.x) * VEC;
      if (col < H) {
        Vec16<T> o, dr;
        if (HAS_DRES) dr.load_nc(dres + base + col);
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float xhat = hv[it].get(i) * rs;
          float v = (dyv[it].get(i) * wv[it].get(i) - xhat * c1) * rs;
          if (HAS_DRES) v += dr.get(i);
          o.set(i, v);
        }
        o.store_na(dx + base + col);
      }
    }
  }
  float* out = dw_partial + (size_t)blockIdx.x * H;
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) out[col + i] = dw_acc[it][i];
    }
  }
}

// out[c] = sum_p partial[p][c]  (coalesced over c; p is small: one per backward CTA)
template <typename T>
__global__ void reduce_partials_kernel(const float* __restrict__ partial, T* __restrict__ out, int P, int H,
                                       int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float s = 0.f;
  for (int p = 0; p < P; ++p) s += partial[(size_t)p * H + c];
  if (accumulate) s += to_f32<T>(out[c]);
  out[c] = from_f32<T>(s);
}

// ------------------------------------------------------------------------------------------- LayerNorm
template <typename T, int MAX_ITERS>
__global__ void __launch_bounds__(1024) layernorm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                             const T* __restrict__ b, T* __restrict__ y,
                                                             float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                             int rows, int H, float eps) {
  constexpr int VEC = Vec16<T>::N;
  __shared__ float red[64];
  const int row = blockIdx.x;
  const size_t base = (size_t)row * H;
  Vec16<T> xv[MAX_ITERS];
  float s[1] = {0.f};
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) {
      xv[it].load_nc(x + base + col);
#pragma unroll
      for (int i = 0; i < VEC; ++i) s[0] += xv[it].get(i);
    }
  }
  block_sum<1>(s, red);
  const float mean = s[0] / (float)H;
  float v[1] = {0.f};
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) { float d = xv[it].get(i) - mean; v[0] += d * d; }
    }
  }
  block_sum<1>(v, red);
  const float rstd = rsqrtf(v[0] / (float)H + eps);
  if (threadIdx.x == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) {
      Vec16<T> wv, bv, o;
      wv.load(w + col);
      if (b) bv.load(b + col);
#pragma unroll
      for (int i = 0; i < VEC; ++i) o.set(i, (xv[it].get(i) - mean) * rstd * wv.get(i) + (b ? bv.get(i) : 0.f));
      o.store_na(y + base + col);
    }
  }
}

template <typename T, int MAX_ITERS>
__global__ void __launch_bounds__(1024) layernorm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                             const T* __restrict__ w, const float* __restrict__ mean,
                                                             const float* __restrict__ rstd, T* __restrict__ dx,
                                                             float* __restrict__ dw_partial,
                                                             float* __restrict__ db_partial, int rows, int H) {
  constexpr int VEC = Vec16<T>::N;
  __shared__ float red[64];
  float dw_acc[MAX_ITERS][VEC], db_acc[MAX_ITERS][VEC];
  Vec16<T> wv[MAX_ITERS];
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) wv[it].load(w + col);
#pragma unroll
    for (int i = 0; i < VEC; ++i) { dw_acc[it][i] = 0.f; db_acc[it][i] = 0.f; }
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const size_t base = (size_t)row * H;
    const float mu = mean[row], rs = rstd[row];
    Vec16<T> dyv[MAX_ITERS], xv[MAX_ITERS];
    float c[2] = {0.f, 0.f};
#pragma unroll
    for (int it = 0; it < MAX_ITERS; ++it) {
      const int col = (it * blockDim.x + threadIdx.x) * VEC;
      if (col < H) {
        dyv[it].load_nc(dy + base + col);
        xv[it].load_nc(x + base + col);
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float xhat = (xv[it].get(i) - mu) * rs, g = dyv[it].get(i), wg = g * wv[it].get(i);
          c[0] += wg;
          c[1] += wg * xhat;
          dw_acc[it][i] += g * xhat;
          db_acc[it][i] += g;
        }
      }
    }
    block_sum<2>(c, red);
    const float c0 = c[0] / (float)H, c1 = c[1] / (float)H;
#pragma unroll
    for (int it = 0; it < MAX_ITERS; ++it) {
      const int col = (it * blockDim.x + threadIdx.x) * VEC;
      if (col < H) {
        Vec16<T> o;
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float xhat = (xv[it].get(i) - mu) * rs;
          o.set(i, (dyv[it].get(i) * wv[it].get(i) - c0 - xhat * c1) * rs);
        }
        o.store_na(dx + base + col);
      }
    }
  }
#pragma unroll
  for (int it = 0; it < MAX_ITERS; ++it) {
    const int col = (it * blockDim.x + threadIdx.x) * VEC;
    if (col < H) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        dw_partial[(size_t)blockIdx.x * H + col + i] = dw_acc[it][i];
        db_partial[(size_t)blockIdx.x * H + col + i] = db_acc[it][i];
      }
    }
  }
}

static inline int pick_block(int H, int vec) {
  int threads = ((H / vec + 31) / 32) * 32;
  if (threads > 1024) threads = 1024;
  if (threads < 32) threads = 32;
  return threads;
}
static inline int pick_iters(int H, int vec, int block) {
  int it = (H / vec + block - 1) / block;
  return it <= 1 ? 1 : (it <= 2 ? 2 : 4);
}
#define CB_DISPATCH_ITERS(iters, IT, ...)            \
  if (iters == 1) { constexpr int IT = 1; __VA_ARGS__; }    \
  else if (iters == 2) { constexpr int IT = 2; __VA_ARGS__; } \
  else { constexpr int IT = 4; __VA_ARGS__; }

extern "C" {

// Max hidden size supported by the register-resident path.
int cb_norm_max_hidden(int dtype) { return 1024 * MAX_ITERS_LIMIT * (dtype == CB_F32 ? 4 : 8); }

int cb_norm_bwd_grid(int rows) {
  int g = cb_num_sms() * 2;
  return rows < g ? rows : g;
}

int cb_rmsnorm_fwd(const void* x, const void* res_in, const void* w, void* y, void* res_out, float* rstd, int rows,
                   int H, float eps, int dtype, cudaStream_t stream) {
  if (rows == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    const int block = pick_block(H, Vec16<T>::N);
    const int iters = pick_iters(H, Vec16<T>::N, block);
    CB_DISPATCH_ITERS(iters, IT, {
      if (res_in)
        rmsnorm_fwd_kernel<T, true, IT><<<rows, block, 0, stream>>>((const T*)x, (const T*)res_in, (const T*)w,
                                                                   (T*)y, (T*)res_out, rstd, rows, H, eps);
      else
        rmsnorm_fwd_kernel<T, false, IT><<<rows, block, 0, stream>>>((const T*)x, nullptr, (const T*)w, (T*)y,
                                                                    nullptr, rstd, rows, H, eps);
    });
  });
  return CB_LAUNCH_CHECK();
}

// dw_partial: fp32 [cb_norm_bwd_grid(rows), H] scratch.  dw: T[H]; accumulate!=0 adds into dw.
int cb_rmsnorm_bwd(const void* dy, const void* h, const void* w, const float* rstd, const void* dres, void* dx,
                   float* dw_partial, void* dw, int accumulate, int rows, int H, int dtype, cudaStream_t stream) {
  if (rows == 0) return 0;
  const int grid = cb_norm_bwd_grid(rows);
  CB_DISPATCH_FLOAT(dtype, T, {
    const int block = pick_block(H, Vec16<T>::N);
    const int iters = pick_iters(H, Vec16<T>::N, block);
    CB_DISPATCH_ITERS(iters, IT, {
      if (dres)
        rmsnorm_bwd_kernel<T, true, IT><<<grid, block, 0, stream>>>((const T*)dy, (const T*)h, (const T*)w, rstd,
                                                                   (const T*)dres, (T*)dx, dw_partial, rows, H);
      else
        rmsnorm_bwd_kernel<T, false, IT><<<grid, block, 0, stream>>>((const T*)dy, (const T*)h, (const T*)w, rstd,
                                                                    nullptr, (T*)dx, dw_partial, rows, H);
    });
    reduce_partials_kernel<T><<<(H + 255) / 256, 256, 0, stream>>>(dw_partial, (T*)dw, grid, H, accumulate);
  });
  return CB_LAUNCH_CHECK();
}

int cb_layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int rows, int H,
                     float eps, int dtype, cudaStream_t stream) {
  if (rows == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    const int block = pick_block(H, Vec16<T>::N);
    const int iters = pick_iters(H, Vec16<T>::N, block);
    CB_DISPATCH_ITERS(iters, IT, {
      layernorm_fwd_kernel<T, IT><<<rows, block, 0, stream>>>((const T*)x, (const T*)w, (const T*)b, (T*)y, mean,
                                                             rstd, rows, H, eps);
    });
  });
  return CB_LAUNCH_CHECK();
}

int cb_layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx,
                     float* dw_partial, float* db_partial, void* dw, void* db, int accumulate, int rows, int H,
                     int dtype, cudaStream_t stream) {
  if (rows == 0) return 0;
  const int grid = cb_norm_bwd_grid(rows);
  CB_DISPATCH_FLOAT(dtype, T, {
    const int block = pick_block(H, Vec16<T>::N);
    const int iters = pick_iters(H, Vec16<T>::N, block);
    CB_DISPATCH_ITERS(iters, IT, {
      layernorm_bwd_kernel<T, IT><<<grid, block, 0, stream>>>((const T*)dy, (const T*)x, (const T*)w, mean, rstd,
                                                             (T*)dx, dw_partial, db_partial, rows, H);
    });
    reduce_partials_kernel<T><<<(H + 255) / 256, 256, 0, stream>>>(dw_partial, (T*)dw, grid, H, accumulate);
    if (db) reduce_partials_kernel<T><<<(H + 255) / 256, 256, 0, stream>>>(db_partial, (T*)db, grid, H, accumulate);
  });
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
