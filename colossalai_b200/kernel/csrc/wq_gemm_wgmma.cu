// Dequantisation of weight-only-quantised linears for sm_90a: the frozen base weights of QLoRA stay packed in HBM, and
// each GEMM that needs one decodes it into a scratch 16-bit weight just before the dense wgmma GEMM (gemm_wgmma.cu)
// consumes it; the scratch is freed when the GEMM is done, so at most one layer's 16-bit weight exists at a time.
//
// Weight formats are the ones quantization/bnb.py stores:
//   4-bit (nf4 / fp4): `packed` uint8, two codes per byte, the high nibble is the even element of the row-major [N, K]
//                      weight; one fp32 absmax per `block_size` consecutive elements (or, with double quantisation, an
//                      int8 absmax_q with absmax = absmax_q * meta[1] + meta[0]); a 16-entry fp32 codebook.
//   int8:              `weight_q` int8 [N, K] with one fp32 scale per output row.
// Every element decodes in fp32 as code[idx] * absmax (or q * scale) and is rounded once to the 16-bit dtype, with
// separately rounded multiplies and adds, so the bytes equal the PyTorch `dequantize()`.
//
// A GEMM that decodes the weight inside its producer warpgroup (no scratch weight) was built and measured on an H100;
// it reached about a third of the throughput of this decode followed by the dense GEMM (docs/kernels.md), because every
// 128-row block of activations decodes the whole weight again, and it was not kept.
#include "common.cuh"

namespace {

enum { WQ_4BIT = 0, WQ_INT8 = 1 };

// The packed weight and its quantisation state.
struct WqWeight {
  const uint8_t* q;         // 4-bit: packed codes (2 per byte); int8: the int8 codes
  const float* absmax;      // 4-bit without double quantisation: one per block; int8: one scale per row
  const int8_t* absmax_q;   // 4-bit with double quantisation (absmax is then null)
  const float* meta;        // [offset, scale] of the double quantisation
  const float* code;        // 16-entry codebook (4-bit)
  int N, K;                 // weight [N, K]
  int block_size;           // 4-bit
};

template <typename T> CB_DEVICE uint32_t pack2(float a, float b);
template <> CB_DEVICE uint32_t pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
template <> CB_DEVICE uint32_t pack2<__half>(float a, float b) {
  __half2 v = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// The absmax of 4-bit block `b`, in fp32 exactly as the PyTorch reference computes it.
CB_DEVICE float block_absmax(const WqWeight& w, int64_t b) {
  if (w.absmax) return __ldg(w.absmax + b);
  return __fadd_rn(__fmul_rn((float)w.absmax_q[b], __ldg(w.meta + 1)), __ldg(w.meta));
}

// 8 consecutive 4-bit codes (4 bytes, the high nibble first) -> 8 elements of T.
template <typename T> CB_DEVICE uint4 decode8_4bit(uint32_t bytes, float absmax, const float* code) {
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t b = (bytes >> (8 * j)) & 0xffu;
    o[j] = pack2<T>(__fmul_rn(code[b >> 4], absmax), __fmul_rn(code[b & 0xfu], absmax));
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

// 8 consecutive int8 codes -> 8 elements of T.
template <typename T> CB_DEVICE uint4 decode8_int8(uint2 bytes, float scale) {
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t w = j < 2 ? bytes.x : bytes.y;
    const int8_t lo = (int8_t)((w >> (16 * (j & 1))) & 0xffu), hi = (int8_t)((w >> (16 * (j & 1) + 8)) & 0xffu);
    o[j] = pack2<T>(__fmul_rn((float)lo, scale), __fmul_rn((float)hi, scale));
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

// ------------------------------------------------------------------------------------------- dequantise to [N, K]
// One thread per group of 8 elements; 4-bit groups never straddle a block (block_size % 8 == 0), int8 groups never
// straddle a row (K % 8 == 0).
template <int FMT, typename T>
__global__ void __launch_bounds__(256) dequant_kernel(const WqWeight w, int64_t numel, T* __restrict__ out) {
  __shared__ float code_s[16];
  if (FMT == WQ_4BIT && threadIdx.x < 16) code_s[threadIdx.x] = w.code[threadIdx.x];
  __syncthreads();
  const int64_t groups = numel / 8;
  for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
    uint4 v;
    if constexpr (FMT == WQ_4BIT) {
      v = decode8_4bit<T>(__ldg(reinterpret_cast<const uint32_t*>(w.q) + g), block_absmax(w, g * 8 / w.block_size),
                          code_s);
    } else {
      v = decode8_int8<T>(__ldg(reinterpret_cast<const uint2*>(w.q) + g), __ldg(w.absmax + g * 8 / w.K));
    }
    reinterpret_cast<uint4*>(out)[g] = v;
  }
}

bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

// Argument checks of the export; fills `w`.
int make_weight(WqWeight& w, int fmt, const void* q, const float* absmax, const int8_t* absmax_q, const float* meta,
                const float* code, int N, int K, int block_size) {
  w = WqWeight{(const uint8_t*)q, absmax, absmax_q, meta, code, N, K, block_size};
  if (N <= 0 || K <= 0 || !aligned16(q) || (K & 7)) return (int)cudaErrorInvalidValue;
  if (fmt == WQ_4BIT) {
    if (!code || (absmax == nullptr) == (absmax_q == nullptr) || (absmax_q && !meta)) return (int)cudaErrorInvalidValue;
    if (block_size <= 0 || (block_size & 7)) return (int)cudaErrorInvalidValue;
  } else if (fmt == WQ_INT8) {
    if (!absmax) return (int)cudaErrorInvalidValue;
  } else {
    return (int)cudaErrorInvalidValue;
  }
  return 0;
}

}  // namespace

extern "C" {

// out[N, K] (bf16 / fp16, 16-byte aligned) = the dequantised weight.  fmt: 0 = 4-bit (absmax or absmax_q + meta, code,
// block_size a multiple of 8; numel = N * K), 1 = int8 (absmax = per-row scales).  N * K must be what the packed buffer
// holds; K must be a multiple of 8.
int cb_wq_dequantize(int fmt, const void* q, const float* absmax, const int8_t* absmax_q, const float* meta,
                     const float* code, int N, int K, int block_size, void* out, int dtype, cudaStream_t stream) {
  WqWeight w;
  int r = make_weight(w, fmt, q, absmax, absmax_q, meta, code, N, K, block_size);
  if (r) return r;
  if (!aligned16(out)) return (int)cudaErrorInvalidValue;
  const int64_t numel = (int64_t)N * K, groups = numel / 8;
  int64_t g = (groups + 255) / 256;
  const int grid = (int)(g < 1 ? 1 : (g > cb_num_sms() * 16 ? cb_num_sms() * 16 : g));
  CB_DISPATCH_HALF(dtype, T, {
    if (fmt == WQ_4BIT) dequant_kernel<WQ_4BIT, T><<<grid, 256, 0, stream>>>(w, numel, (T*)out);
    else dequant_kernel<WQ_INT8, T><<<grid, 256, 0, stream>>>(w, numel, (T*)out);
  });
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
