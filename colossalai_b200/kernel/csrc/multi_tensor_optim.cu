// Multi-tensor optimizer kernels for sm_90a: Adam/AdamW (fp32 master + low-precision working copy written in the
// same pass, fused grad un-scale / clip), SGD(+momentum, nesterov), LAMB (two stages), L2/max norm, scale+inf check.
//
// Capability parity: reference fused_optim_cuda (extensions/csrc/kernel/cuda/multi_tensor_{adam,sgd,lamb,l2norm,
// scale}_kernel.cu, N3-N7) and its apex-derived multi_tensor_apply.cuh harness.  Design is new: instead of packing
// <=36 tensor pointers into kernel arguments and launching many times, ONE device-resident descriptor table
// (built once per parameter group and cached) describes every tensor; a single launch covers the whole group and
// each CTA binary-searches its (tensor, chunk) from a chunk-prefix array.  All kernels are HBM-bound streaming
// passes with 16-byte vector accesses.
#include "common.cuh"

// One row per tensor, 8 x int64:  [0] param ptr  [1] grad ptr  [2] exp_avg ptr  [3] exp_avg_sq ptr
//                                  [4] low-precision copy ptr (or 0)  [5] numel
//                                  [6] dtype codes packed: param | grad<<8 | lp<<16   [7] chunk prefix (exclusive)
constexpr int TBL_COLS = 8;
constexpr int CHUNK = 2048 * 16;   // elements per CTA work item
constexpr int OPT_THREADS = 512;

struct TensorRef {
  void *p, *g, *m, *v, *lp;
  int64_t n;
  int pd, gd, ld;
  int64_t chunk0;
};

CB_DEVICE TensorRef load_ref(const int64_t* tbl, int t) {
  const int64_t* r = tbl + (int64_t)t * TBL_COLS;
  TensorRef x;
  x.p = (void*)r[0]; x.g = (void*)r[1]; x.m = (void*)r[2]; x.v = (void*)r[3]; x.lp = (void*)r[4];
  x.n = r[5];
  x.pd = (int)(r[6] & 0xff); x.gd = (int)((r[6] >> 8) & 0xff); x.ld = (int)((r[6] >> 16) & 0xff);
  x.chunk0 = r[7];
  return x;
}

// largest t with chunk_prefix[t] <= chunk
CB_DEVICE int find_tensor(const int64_t* tbl, int num_tensors, int64_t chunk) {
  int lo = 0, hi = num_tensors - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tbl[(int64_t)mid * TBL_COLS + 7] <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

CB_DEVICE float ld_any(const void* p, int dt, int64_t i) {
  switch (dt) {
    case CB_F32: return ((const float*)p)[i];
    case CB_F16: return __half2float(((const __half*)p)[i]);
    default: return __bfloat162float(((const __nv_bfloat16*)p)[i]);
  }
}
CB_DEVICE void st_any(void* p, int dt, int64_t i, float v) {
  switch (dt) {
    case CB_F32: ((float*)p)[i] = v; break;
    case CB_F16: ((__half*)p)[i] = __float2half_rn(v); break;
    default: ((__nv_bfloat16*)p)[i] = __float2bfloat16_rn(v); break;
  }
}

struct AdamHyper {
  float lr, beta1, beta2, eps, weight_decay, bc1, bc2, inv_scale;
  int adamw;  // 1 = decoupled weight decay
};

// Vectorised fast path: fp32 param/m/v, TG grad, TL low-precision copy (or none), 4 elements per thread-iteration.
template <typename TG, typename TL, bool HAS_LP>
CB_DEVICE void adam_chunk_vec(float* __restrict__ p, const TG* __restrict__ g, float* __restrict__ m,
                              float* __restrict__ v, TL* __restrict__ lp, int64_t n, const AdamHyper h) {
  for (int64_t i = (int64_t)threadIdx.x * 4; i < n; i += (int64_t)blockDim.x * 4) {
    float pv[4], gv[4], mv[4], vv[4];
    if (i + 3 < n) {
      const float4 p4 = *reinterpret_cast<const float4*>(p + i);
      const float4 m4 = *reinterpret_cast<const float4*>(m + i);
      const float4 v4 = *reinterpret_cast<const float4*>(v + i);
      pv[0] = p4.x; pv[1] = p4.y; pv[2] = p4.z; pv[3] = p4.w;
      mv[0] = m4.x; mv[1] = m4.y; mv[2] = m4.z; mv[3] = m4.w;
      vv[0] = v4.x; vv[1] = v4.y; vv[2] = v4.z; vv[3] = v4.w;
#pragma unroll
      for (int k = 0; k < 4; ++k) gv[k] = to_f32<TG>(g[i + k]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float gg = gv[k] * h.inv_scale;
        if (!h.adamw) gg += h.weight_decay * pv[k];
        mv[k] = h.beta1 * mv[k] + (1.f - h.beta1) * gg;
        vv[k] = h.beta2 * vv[k] + (1.f - h.beta2) * gg * gg;
        float upd = (mv[k] / h.bc1) / (sqrtf(vv[k] / h.bc2) + h.eps);
        if (h.adamw) upd += h.weight_decay * pv[k];
        pv[k] -= h.lr * upd;
      }
      *reinterpret_cast<float4*>(p + i) = make_float4(pv[0], pv[1], pv[2], pv[3]);
      *reinterpret_cast<float4*>(m + i) = make_float4(mv[0], mv[1], mv[2], mv[3]);
      *reinterpret_cast<float4*>(v + i) = make_float4(vv[0], vv[1], vv[2], vv[3]);
      if (HAS_LP) {
#pragma unroll
        for (int k = 0; k < 4; ++k) lp[i + k] = from_f32<TL>(pv[k]);
      }
    } else {
      for (int64_t j = i; j < n; ++j) {
        float pp = p[j], gg = to_f32<TG>(g[j]) * h.inv_scale, mm = m[j], vx = v[j];
        if (!h.adamw) gg += h.weight_decay * pp;
        mm = h.beta1 * mm + (1.f - h.beta1) * gg;
        vx = h.beta2 * vx + (1.f - h.beta2) * gg * gg;
        float upd = (mm / h.bc1) / (sqrtf(vx / h.bc2) + h.eps);
        if (h.adamw) upd += h.weight_decay * pp;
        pp -= h.lr * upd;
        p[j] = pp; m[j] = mm; v[j] = vx;
        if (HAS_LP) lp[j] = from_f32<TL>(pp);
      }
    }
  }
}

CB_DEVICE void adam_chunk_generic(const TensorRef& t, int64_t off, int64_t n, const AdamHyper h) {
  float* m = (float*)t.m + off;
  float* v = (float*)t.v + off;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
    float pp = ld_any(t.p, t.pd, off + j), gg = ld_any(t.g, t.gd, off + j) * h.inv_scale, mm = m[j], vx = v[j];
    if (!h.adamw) gg += h.weight_decay * pp;
    mm = h.beta1 * mm + (1.f - h.beta1) * gg;
    vx = h.beta2 * vx + (1.f - h.beta2) * gg * gg;
    float upd = (mm / h.bc1) / (sqrtf(vx / h.bc2) + h.eps);
    if (h.adamw) upd += h.weight_decay * pp;
    pp -= h.lr * upd;
    st_any(t.p, t.pd, off + j, pp);
    m[j] = mm; v[j] = vx;
    if (t.lp) st_any(t.lp, t.ld, off + j, pp);
  }
}

__global__ void __launch_bounds__(OPT_THREADS) multi_tensor_adam_kernel(const int64_t* __restrict__ tbl,
                                                                        int num_tensors, AdamHyper h,
                                                                        const int* __restrict__ noop_flag,
                                                                        const float* __restrict__ inv_scale_dev) {
  if (noop_flag && *noop_flag) return;
  if (inv_scale_dev) h.inv_scale *= *inv_scale_dev;   // device-resident clip/unscale coefficient (no host sync)
  const int64_t chunk = blockIdx.x;
  const int ti = find_tensor(tbl, num_tensors, chunk);
  const TensorRef t = load_ref(tbl, ti);
  const int64_t off = (chunk - t.chunk0) * CHUNK;
  if (off >= t.n) return;
  const int64_t n = min((int64_t)CHUNK, t.n - off);
  const bool aligned = ((((uintptr_t)t.p) | ((uintptr_t)t.m) | ((uintptr_t)t.v)) & 15) == 0;
  if (t.pd == CB_F32 && aligned) {
    float* p = (float*)t.p + off; float* m = (float*)t.m + off; float* v = (float*)t.v + off;
#define ADAM_CASE(TG, TL, HAS)                                                                    \
    adam_chunk_vec<TG, TL, HAS>(p, (const TG*)t.g + off, m, v, (TL*)t.lp + (HAS ? off : 0), n, h)
    if (t.gd == CB_BF16) {
      if (t.lp && t.ld == CB_BF16) ADAM_CASE(__nv_bfloat16, __nv_bfloat16, true);
      else if (!t.lp) ADAM_CASE(__nv_bfloat16, __nv_bfloat16, false);
      else adam_chunk_generic(t, off, n, h);
    } else if (t.gd == CB_F32) {
      if (t.lp && t.ld == CB_BF16) ADAM_CASE(float, __nv_bfloat16, true);
      else if (t.lp && t.ld == CB_F16) ADAM_CASE(float, __half, true);
      else if (!t.lp) ADAM_CASE(float, float, false);
      else adam_chunk_generic(t, off, n, h);
    } else if (t.gd == CB_F16) {
      if (t.lp && t.ld == CB_F16) ADAM_CASE(__half, __half, true);
      else if (!t.lp) ADAM_CASE(__half, __half, false);
      else adam_chunk_generic(t, off, n, h);
    } else {
      adam_chunk_generic(t, off, n, h);
    }
#undef ADAM_CASE
  } else {
    adam_chunk_generic(t, off, n, h);
  }
}

// ------------------------------------------------------------------------------------------------ SGD
struct SgdHyper { float lr, momentum, dampening, weight_decay, inv_scale; int nesterov, first_run, wd_after; };

__global__ void __launch_bounds__(OPT_THREADS) multi_tensor_sgd_kernel(const int64_t* __restrict__ tbl,
                                                                       int num_tensors, SgdHyper h,
                                                                       const int* __restrict__ noop_flag) {
  if (noop_flag && *noop_flag) return;
  const int64_t chunk = blockIdx.x;
  const TensorRef t = load_ref(tbl, find_tensor(tbl, num_tensors, chunk));
  const int64_t off = (chunk - t.chunk0) * CHUNK;
  if (off >= t.n) return;
  const int64_t n = min((int64_t)CHUNK, t.n - off);
  float* mom = t.m ? (float*)t.m + off : nullptr;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
    float p = ld_any(t.p, t.pd, off + j), g = ld_any(t.g, t.gd, off + j) * h.inv_scale;
    if (h.weight_decay != 0.f && !h.wd_after) g += h.weight_decay * p;
    if (h.momentum != 0.f && mom) {
      float b = h.first_run ? g : mom[j] * h.momentum + (1.f - h.dampening) * g;
      mom[j] = b;
      g = h.nesterov ? g + h.momentum * b : b;
    }
    if (h.weight_decay != 0.f && h.wd_after) g += h.weight_decay * p;
    p -= h.lr * g;
    st_any(t.p, t.pd, off + j, p);
    if (t.lp) st_any(t.lp, t.ld, off + j, p);
  }
}

// ------------------------------------------------------------------------------------------------ norms
// The max norm propagates NaN like torch's `vector_norm(ord=inf)`: `fmaxf` (PTX `max.f32`) returns the other
// operand when one is NaN, so a NaN gradient would report a finite norm.  `max.NaN.f32` (sm_80+) returns NaN.
CB_DEVICE float nan_max(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

CB_DEVICE float block_max_nan(float v, float* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (nwarps == 1) return v;
  __syncthreads();
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  v = lane < nwarps ? smem[lane] : 0.f;   // every partial is an absolute value (>= 0) or NaN
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// partial[chunk] = sum (or max) over the chunk of x^2 (|x|); `which`: 0 = param, 1 = grad, 2 = m (update buffer)
__global__ void __launch_bounds__(OPT_THREADS) multi_tensor_norm_partial_kernel(const int64_t* __restrict__ tbl,
                                                                               int num_tensors, int which,
                                                                               int use_max,
                                                                               float* __restrict__ partial) {
  __shared__ float red[64];
  const int64_t chunk = blockIdx.x;
  const TensorRef t = load_ref(tbl, find_tensor(tbl, num_tensors, chunk));
  const int64_t off = (chunk - t.chunk0) * CHUNK;
  float acc = 0.f;
  if (off < t.n) {
    const int64_t n = min((int64_t)CHUNK, t.n - off);
    const void* src = which == 0 ? t.p : (which == 1 ? t.g : t.m);
    const int dt = which == 0 ? t.pd : (which == 1 ? t.gd : CB_F32);
    const int esz = dt == CB_F32 ? 4 : 2;
    const char* base = reinterpret_cast<const char*>(src) + off * esz;
    const int per = 16 / esz;                                   // elements per 16-byte vector
    int64_t head = 0;                                           // scalar prologue up to 16-byte alignment
    const uintptr_t mis = reinterpret_cast<uintptr_t>(base) & 15;
    if (mis) head = min(n, (int64_t)((16 - mis) / esz));
    for (int64_t j = threadIdx.x; j < head; j += blockDim.x) {
      const float x = ld_any(src, dt, off + j);
      acc = use_max ? nan_max(acc, fabsf(x)) : acc + x * x;
    }
    const int64_t nvec = (n - head) / per;
    const uint4* vp = reinterpret_cast<const uint4*>(base + head * esz);
    float acc2 = 0.f;                                           // two accumulators: more loads in flight
    for (int64_t j = threadIdx.x; j < nvec; j += 2 * blockDim.x) {
      uint4 r0, r1 = make_uint4(0, 0, 0, 0);
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                   : "=r"(r0.x), "=r"(r0.y), "=r"(r0.z), "=r"(r0.w) : "l"(vp + j));
      const bool two = j + blockDim.x < nvec;
      if (two)
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(r1.x), "=r"(r1.y), "=r"(r1.z), "=r"(r1.w) : "l"(vp + j + blockDim.x));
      const uint32_t w0[4] = {r0.x, r0.y, r0.z, r0.w};
      const uint32_t w1[4] = {r1.x, r1.y, r1.z, r1.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float a0, a1, b0, b1;
        if (dt == CB_F32) {
          a0 = __uint_as_float(w0[q]); a1 = 0.f; b0 = __uint_as_float(w1[q]); b1 = 0.f;
        } else if (dt == CB_BF16) {
          a0 = __uint_as_float(w0[q] << 16); a1 = __uint_as_float(w0[q] & 0xffff0000u);
          b0 = __uint_as_float(w1[q] << 16); b1 = __uint_as_float(w1[q] & 0xffff0000u);
        } else {
          const __half2 h0 = *reinterpret_cast<const __half2*>(&w0[q]);
          const __half2 h1 = *reinterpret_cast<const __half2*>(&w1[q]);
          a0 = __low2float(h0); a1 = __high2float(h0); b0 = __low2float(h1); b1 = __high2float(h1);
        }
        if (use_max) {
          acc = nan_max(acc, nan_max(fabsf(a0), fabsf(a1)));
          acc2 = nan_max(acc2, nan_max(fabsf(b0), fabsf(b1)));
        } else {
          acc += a0 * a0 + a1 * a1;
          acc2 += b0 * b0 + b1 * b1;
        }
      }
    }
    acc = use_max ? nan_max(acc, acc2) : acc + acc2;
    for (int64_t j = head + nvec * per + threadIdx.x; j < n; j += blockDim.x) {     // scalar tail
      const float x = ld_any(src, dt, off + j);
      acc = use_max ? nan_max(acc, fabsf(x)) : acc + x * x;
    }
  }
  if (use_max) {
    acc = block_max_nan(acc, red);
  } else {
    float a[1] = {acc};
    block_sum<1>(a, red);
    acc = a[0];
  }
  if (threadIdx.x == 0) partial[chunk] = acc;
}

// out[0] = reduce(partial[0..n)) ; per_tensor[t] = reduce over that tensor's chunks (optional)
__global__ void __launch_bounds__(1024) norm_finalize_kernel(const float* __restrict__ partial, int64_t n_chunks,
                                                             const int64_t* __restrict__ tbl, int num_tensors,
                                                             int use_max, float* __restrict__ out,
                                                             float* __restrict__ per_tensor) {
  __shared__ float red[64];
  if (blockIdx.x == 0) {
    float acc = 0.f;
    for (int64_t i = threadIdx.x; i < n_chunks; i += blockDim.x)
      acc = use_max ? nan_max(acc, partial[i]) : acc + partial[i];
    if (use_max) acc = block_max_nan(acc, red);
    else { float a[1] = {acc}; block_sum<1>(a, red); acc = a[0]; }
    if (threadIdx.x == 0) out[0] = acc;   // squared L2 norm (or max): python takes the sqrt after cross-rank reduce
  } else if (per_tensor) {
    for (int t = blockIdx.x - 1; t < num_tensors; t += gridDim.x - 1) {
      const int64_t c0 = tbl[(int64_t)t * TBL_COLS + 7];
      const int64_t c1 = (t + 1 < num_tensors) ? tbl[(int64_t)(t + 1) * TBL_COLS + 7] : n_chunks;
      float acc = 0.f;
      for (int64_t i = c0 + threadIdx.x; i < c1; i += blockDim.x)
        acc = use_max ? nan_max(acc, partial[i]) : acc + partial[i];
      if (use_max) acc = block_max_nan(acc, red);
      else { float a[1] = {acc}; block_sum<1>(a, red); acc = a[0]; }
      if (threadIdx.x == 0) per_tensor[t] = acc;
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------------ scale
// dst(grad slot) = src(param slot) * scale, flag on inf/nan.  Table: param = src, grad = dst.
__global__ void __launch_bounds__(OPT_THREADS) multi_tensor_scale_kernel(const int64_t* __restrict__ tbl,
                                                                         int num_tensors, float scale,
                                                                         int* __restrict__ flag) {
  const int64_t chunk = blockIdx.x;
  const TensorRef t = load_ref(tbl, find_tensor(tbl, num_tensors, chunk));
  const int64_t off = (chunk - t.chunk0) * CHUNK;
  if (off >= t.n) return;
  const int64_t n = min((int64_t)CHUNK, t.n - off);
  bool bad = false;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
    const float x = ld_any(t.p, t.pd, off + j);
    if (!isfinite(x)) bad = true;
    st_any(t.g, t.gd, off + j, x * scale);
  }
  if (flag && __any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) *flag = 1;
}

// ------------------------------------------------------------------------------------------------ LAMB
// stage 1: m, v update; "update" u = m_hat / (sqrt(v_hat) + eps) + wd * p is written into the GRAD slot (in place).
struct LambHyper { float beta1, beta2, beta3, eps, weight_decay, bc1, bc2, inv_scale, lr; int adamw; };

__global__ void __launch_bounds__(OPT_THREADS) multi_tensor_lamb_stage1_kernel(const int64_t* __restrict__ tbl,
                                                                               int num_tensors, LambHyper h,
                                                                               const int* __restrict__ noop_flag) {
  if (noop_flag && *noop_flag) return;
  const int64_t chunk = blockIdx.x;
  const TensorRef t = load_ref(tbl, find_tensor(tbl, num_tensors, chunk));
  const int64_t off = (chunk - t.chunk0) * CHUNK;
  if (off >= t.n) return;
  const int64_t n = min((int64_t)CHUNK, t.n - off);
  float* m = (float*)t.m + off; float* v = (float*)t.v + off;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
    const float p = ld_any(t.p, t.pd, off + j);
    float g = ld_any(t.g, t.gd, off + j) * h.inv_scale;
    if (!h.adamw) g += h.weight_decay * p;
    const float mm = h.beta1 * m[j] + h.beta3 * g;
    const float vx = h.beta2 * v[j] + (1.f - h.beta2) * g * g;
    m[j] = mm; v[j] = vx;
    float u = (mm / h.bc1) / (sqrtf(vx / h.bc2) + h.eps);
    if (h.adamw) u += h.weight_decay * p;
    st_any(t.g, t.gd, off + j, u);
  }
}

// stage 2: p -= lr * trust_ratio[t] * u   with trust = ||p|| / ||u|| (1 when either is 0).  Null norm pointers mean
// no trust ratio (ratio 1): the reference applies it only with `use_nvlamb` or a non-zero weight decay.
__global__ void __launch_bounds__(OPT_THREADS) multi_tensor_lamb_stage2_kernel(const int64_t* __restrict__ tbl,
                                                                               int num_tensors, float lr,
                                                                               const float* __restrict__ p_norm_sq,
                                                                               const float* __restrict__ u_norm_sq,
                                                                               const int* __restrict__ noop_flag) {
  if (noop_flag && *noop_flag) return;
  const int64_t chunk = blockIdx.x;
  const int ti = find_tensor(tbl, num_tensors, chunk);
  const TensorRef t = load_ref(tbl, ti);
  const int64_t off = (chunk - t.chunk0) * CHUNK;
  if (off >= t.n) return;
  const int64_t n = min((int64_t)CHUNK, t.n - off);
  float ratio = 1.f;
  if (p_norm_sq && u_norm_sq) {
    const float pn = sqrtf(p_norm_sq[ti]), un = sqrtf(u_norm_sq[ti]);
    if (pn > 0.f && un > 0.f) ratio = pn / un;
  }
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
    float p = ld_any(t.p, t.pd, off + j);
    p -= lr * ratio * ld_any(t.g, t.gd, off + j);
    st_any(t.p, t.pd, off + j, p);
    if (t.lp) st_any(t.lp, t.ld, off + j, p);
  }
}

extern "C" {

int cb_opt_chunk_size() { return CHUNK; }
int cb_opt_table_cols() { return TBL_COLS; }

int cb_multi_tensor_adam(const int64_t* tbl, int num_tensors, int64_t total_chunks, float lr, float beta1, float beta2,
                         float eps, float weight_decay, float bc1, float bc2, float inv_scale, int adamw,
                         const int* noop_flag, const float* inv_scale_dev, cudaStream_t s) {
  if (total_chunks == 0) return 0;
  AdamHyper h{lr, beta1, beta2, eps, weight_decay, bc1, bc2, inv_scale, adamw};
  multi_tensor_adam_kernel<<<(unsigned)total_chunks, OPT_THREADS, 0, s>>>(tbl, num_tensors, h, noop_flag,
                                                                          inv_scale_dev);
  return CB_LAUNCH_CHECK();
}

int cb_multi_tensor_sgd(const int64_t* tbl, int num_tensors, int64_t total_chunks, float lr, float momentum,
                        float dampening, float weight_decay, float inv_scale, int nesterov, int first_run,
                        int wd_after, const int* noop_flag, cudaStream_t s) {
  if (total_chunks == 0) return 0;
  SgdHyper h{lr, momentum, dampening, weight_decay, inv_scale, nesterov, first_run, wd_after};
  multi_tensor_sgd_kernel<<<(unsigned)total_chunks, OPT_THREADS, 0, s>>>(tbl, num_tensors, h, noop_flag);
  return CB_LAUNCH_CHECK();
}

// out[0] = sum of squares (or max abs) over all tensors; per_tensor (optional) [num_tensors]; partial: [total_chunks]
int cb_multi_tensor_norm(const int64_t* tbl, int num_tensors, int64_t total_chunks, int which, int use_max,
                         float* partial, float* out, float* per_tensor, cudaStream_t s) {
  if (total_chunks == 0) { cudaMemsetAsync(out, 0, sizeof(float), s); return 0; }
  multi_tensor_norm_partial_kernel<<<(unsigned)total_chunks, OPT_THREADS, 0, s>>>(tbl, num_tensors, which, use_max,
                                                                                  partial);
  int blocks = 1;
  if (per_tensor) { blocks += num_tensors < 1024 ? num_tensors : 1024; }
  norm_finalize_kernel<<<blocks, 1024, 0, s>>>(partial, total_chunks, tbl, num_tensors, use_max, out, per_tensor);
  return CB_LAUNCH_CHECK();
}

int cb_multi_tensor_scale(const int64_t* tbl, int num_tensors, int64_t total_chunks, float scale, int* flag,
                          cudaStream_t s) {
  if (total_chunks == 0) return 0;
  multi_tensor_scale_kernel<<<(unsigned)total_chunks, OPT_THREADS, 0, s>>>(tbl, num_tensors, scale, flag);
  return CB_LAUNCH_CHECK();
}

int cb_multi_tensor_lamb_stage1(const int64_t* tbl, int num_tensors, int64_t total_chunks, float beta1, float beta2,
                                float beta3, float eps, float weight_decay, float bc1, float bc2, float inv_scale,
                                int adamw, const int* noop_flag, cudaStream_t s) {
  if (total_chunks == 0) return 0;
  LambHyper h{beta1, beta2, beta3, eps, weight_decay, bc1, bc2, inv_scale, 0.f, adamw};
  multi_tensor_lamb_stage1_kernel<<<(unsigned)total_chunks, OPT_THREADS, 0, s>>>(tbl, num_tensors, h, noop_flag);
  return CB_LAUNCH_CHECK();
}

int cb_multi_tensor_lamb_stage2(const int64_t* tbl, int num_tensors, int64_t total_chunks, float lr,
                                const float* p_norm_sq, const float* u_norm_sq, const int* noop_flag,
                                cudaStream_t s) {
  if (total_chunks == 0) return 0;
  multi_tensor_lamb_stage2_kernel<<<(unsigned)total_chunks, OPT_THREADS, 0, s>>>(tbl, num_tensors, lr, p_norm_sq,
                                                                                 u_norm_sq, noop_flag);
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
