// Host-side Adam/AdamW for Gemini-offloaded optimizer shards (pinned host memory).
//
// Capability parity: reference cpu_adam_x86 / cpu_adam_arm (extensions/csrc/kernel/{x86,arm}/cpu_adam*.cpp, N1/N2):
// fp32/fp16 params & grads, fused grad un-scale, both weight-decay modes.  New here: bf16 params/grads are handled
// natively (the reference falls back to torch ops for bf16, nn/optimizer/hybrid_adam.py:126-143), an optional
// low-precision copy of the updated parameter is written in the same pass (saves one full re-read before the H2D
// upload), and ISA dispatch happens at RUN time (target_clones: AVX-512 / AVX2 / scalar) so a library built on one
// host runs on another.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <omp.h>

namespace {

inline float bf16_to_f32(uint16_t v) {
  uint32_t u = (uint32_t)v << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
inline uint16_t f32_to_bf16(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
  u += 0x7fffu + ((u >> 16) & 1u);                                            // round to nearest even
  return (uint16_t)(u >> 16);
}
inline float f16_to_f32(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1fu, man = h & 0x3ffu, u;
  if (exp == 0) {
    if (man == 0) u = sign;
    else {
      exp = 127 - 15 + 1;
      while (!(man & 0x400u)) { man <<= 1; --exp; }
      man &= 0x3ffu;
      u = sign | (exp << 23) | (man << 13);
    }
  } else if (exp == 31) u = sign | 0x7f800000u | (man << 13);
  else u = sign | ((exp + 127 - 15) << 23) | (man << 13);
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
inline uint16_t f32_to_f16(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  const uint32_t sign = (u >> 16) & 0x8000u;
  int32_t exp = (int32_t)((u >> 23) & 0xff) - 127 + 15;
  uint32_t man = u & 0x7fffffu;
  if (((u >> 23) & 0xff) == 0xff) return (uint16_t)(sign | 0x7c00u | (man ? 0x200u : 0));
  if (exp >= 31) return (uint16_t)(sign | 0x7c00u);
  // round to nearest, ties to even (a carry out of the mantissa bumps the exponent, up to inf)
  if (exp <= 0) {
    if (exp < -10) return (uint16_t)sign;
    man |= 0x800000u;
    const int shift = 14 - exp;
    uint32_t r = man >> shift;
    const uint32_t rem = man & ((1u << shift) - 1u), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (r & 1u))) r += 1;
    return (uint16_t)(sign | r);
  }
  uint32_t r = (uint32_t)(exp << 10) | (man >> 13);
  const uint32_t rem = man & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (r & 1u))) r += 1;
  return (uint16_t)(sign | r);
}

// dtype codes: 0 f32, 1 f16, 2 bf16  (same as the CUDA side)
template <int DT> inline float ld(const void* p, int64_t i);
template <> inline float ld<0>(const void* p, int64_t i) { return ((const float*)p)[i]; }
template <> inline float ld<1>(const void* p, int64_t i) { return f16_to_f32(((const uint16_t*)p)[i]); }
template <> inline float ld<2>(const void* p, int64_t i) { return bf16_to_f32(((const uint16_t*)p)[i]); }
template <int DT> inline void st(void* p, int64_t i, float v);
template <> inline void st<0>(void* p, int64_t i, float v) { ((float*)p)[i] = v; }
template <> inline void st<1>(void* p, int64_t i, float v) { ((uint16_t*)p)[i] = f32_to_f16(v); }
template <> inline void st<2>(void* p, int64_t i, float v) { ((uint16_t*)p)[i] = f32_to_bf16(v); }

struct Hyper {
  float lr, beta1, beta2, eps, wd, bc1, bc2, inv_scale;
  int adamw;
};

template <int PD, int GD, int LD>
__attribute__((target_clones("arch=skylake-avx512", "avx2", "default")))
void adam_block(void* p, const void* g, float* m, float* v, void* lp, int64_t s, int64_t e, Hyper h) {
  const float ob1 = 1.f - h.beta1, ob2 = 1.f - h.beta2, ibc1 = 1.f / h.bc1, ibc2 = 1.f / h.bc2;
#pragma GCC ivdep
  for (int64_t i = s; i < e; ++i) {
    float pp = ld<PD>(p, i);
    float gg = ld<GD>(g, i) * h.inv_scale;
    if (!h.adamw) gg += h.wd * pp;
    const float mm = h.beta1 * m[i] + ob1 * gg;
    const float vv = h.beta2 * v[i] + ob2 * gg * gg;
    m[i] = mm;
    v[i] = vv;
    float upd = (mm * ibc1) / (std::sqrt(vv * ibc2) + h.eps);
    if (h.adamw) upd += h.wd * pp;
    pp -= h.lr * upd;
    st<PD>(p, i, pp);
    if (LD >= 0) st<(LD >= 0 ? LD : 0)>(lp, i, pp);
  }
}

template <int PD, int GD, int LD>
void adam_span(void* p, const void* g, float* m, float* v, void* lp, int64_t n, Hyper h) {
  const int64_t BLK = 8192;
#pragma omp parallel for schedule(static)
  for (int64_t blk = 0; blk < (n + BLK - 1) / BLK; ++blk) {
    const int64_t s = blk * BLK, e = s + BLK < n ? s + BLK : n;
    adam_block<PD, GD, LD>(p, g, m, v, lp, s, e, h);
  }
}

template <int PD, int GD>
void dispatch_lp(void* p, const void* g, float* m, float* v, void* lp, int lpd, int64_t n, Hyper h) {
  if (!lp) adam_span<PD, GD, -1>(p, g, m, v, nullptr, n, h);
  else if (lpd == 2) adam_span<PD, GD, 2>(p, g, m, v, lp, n, h);
  else if (lpd == 1) adam_span<PD, GD, 1>(p, g, m, v, lp, n, h);
  else adam_span<PD, GD, 0>(p, g, m, v, lp, n, h);
}

template <int PD>
void dispatch_g(void* p, const void* g, int gd, float* m, float* v, void* lp, int lpd, int64_t n, Hyper h) {
  if (gd == 0) dispatch_lp<PD, 0>(p, g, m, v, lp, lpd, n, h);
  else if (gd == 1) dispatch_lp<PD, 1>(p, g, m, v, lp, lpd, n, h);
  else dispatch_lp<PD, 2>(p, g, m, v, lp, lpd, n, h);
}

}  // namespace

extern "C" {

// Returns 0 on success.  `lp` may be null.  exp_avg / exp_avg_sq are always fp32.
int cb_cpu_adam_step(void* p, int pd, const void* g, int gd, float* exp_avg, float* exp_avg_sq, void* lp, int lpd,
                     int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                     int bias_correction, int adamw, float inv_scale) {
  Hyper h;
  h.lr = lr; h.beta1 = beta1; h.beta2 = beta2; h.eps = eps; h.wd = weight_decay; h.inv_scale = inv_scale;
  h.adamw = adamw;
  h.bc1 = bias_correction ? 1.f - std::pow(beta1, (float)step) : 1.f;
  h.bc2 = bias_correction ? 1.f - std::pow(beta2, (float)step) : 1.f;
  if (pd == 0) dispatch_g<0>(p, g, gd, exp_avg, exp_avg_sq, lp, lpd, n, h);
  else if (pd == 1) dispatch_g<1>(p, g, gd, exp_avg, exp_avg_sq, lp, lpd, n, h);
  else if (pd == 2) dispatch_g<2>(p, g, gd, exp_avg, exp_avg_sq, lp, lpd, n, h);
  else return 1;
  return 0;
}

// sum of squares of a host buffer (grad-norm of offloaded shards)
double cb_cpu_sumsq(const void* x, int dt, int64_t n) {
  double acc = 0.0;
#pragma omp parallel for reduction(+ : acc) schedule(static)
  for (int64_t i = 0; i < n; ++i) {
    const float f = dt == 0 ? ((const float*)x)[i] : (dt == 1 ? f16_to_f32(((const uint16_t*)x)[i])
                                                              : bf16_to_f32(((const uint16_t*)x)[i]));
    acc += (double)f * (double)f;
  }
  return acc;
}

int cb_cpu_num_threads() { return omp_get_max_threads(); }

const char* cb_cpu_isa() {
  __builtin_cpu_init();
  if (__builtin_cpu_supports("avx512f")) return "avx512";
  if (__builtin_cpu_supports("avx2")) return "avx2";
  return "scalar";
}

}  // extern "C"
