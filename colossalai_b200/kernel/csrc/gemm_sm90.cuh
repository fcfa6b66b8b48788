// Warp-specialised wgmma GEMM main loop for sm_90a, shared by the dense (gemm_wgmma.cu), grouped (grouped_gemm_wgmma.cu)
// and comm-fused (fused_comm_gemm.cu) GEMMs:  D[128 x 128 tile] (+)= sum_k A(m, k) * B(n, k), fp32 accumulate (int32 for
// the int8 W8A8 GEMM).
//
//   * operands are staged by TMA (cp.async.bulk.tensor, SWIZZLE_128B) through a STAGES-deep mbarrier ring by one
//     producer warp (warp 8);
//   * two consumer warpgroups (warps 0..7) each own 64 rows of the tile and issue wgmma m64n128k16 (16-bit operands) or
//     m64n128k32 (8-bit float or int8 operands) straight from shared memory; the accumulator lives in registers
//     (64 / thread);
//   * a stage is handed back to the producer as soon as the wgmma group reading it has retired (one group in flight);
//   * A and B may each be K-major ("row = M/N, contiguous K") or MN-major ("row = K, contiguous M/N", 16-bit only),
//     which covers the three GEMMs of a linear layer without any transposition pass;
//   * the kernel is persistent: CTA b walks tiles b, b + grid, ...; the producer runs ahead into the next tile while the
//     consumers store the previous one.
// A problem type `Prob` maps a tile index to operand coordinates and an output window; it may also provide hooks
// (`before_load`: the producer waits for its operands to exist, `after_store`: a consumer warpgroup publishes a tile).
#pragma once
#include "common.cuh"
#include "sm90.cuh"

#include <type_traits>

namespace gemm90 {
using namespace sm90;

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int KBYTES = 128;                 // bytes of K per stage and row: 64 x 16-bit or 128 x 8-bit
constexpr int STAGES = 6;
constexpr int A_BYTES = BM * KBYTES;        // 16 KB
constexpr int B_BYTES = BN * KBYTES;        // 16 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int CONSUMER_THREADS = 256;
constexpr int PRODUCER_WARP = 8;
constexpr int NUM_THREADS = CONSUMER_THREADS + 32;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int GROUP_M = 8;

// element kinds of the operands
enum { K_BF16 = 0, K_F16 = 1, K_E4M3_E4M3 = 2, K_E4M3_E5M2 = 3, K_E5M2_E4M3 = 4, K_E5M2_E5M2 = 5, K_S8 = 6 };
template <int KIND> struct KindTraits {
  static constexpr bool F8 = KIND >= K_E4M3_E4M3 && KIND <= K_E5M2_E5M2;
  static constexpr bool S8 = KIND == K_S8;
  static constexpr int KE = F8 || S8 ? 128 : 64;    // K elements per stage
  static constexpr int MMA_K = F8 || S8 ? 32 : 16;  // K elements per instruction (32 bytes either way)
  // int8 products are summed exactly in int32 (|acc| <= 127 * 127 * K: the launcher bounds K)
  using Acc = typename std::conditional<S8, int, float>::type;
};

// One tile of work: operand coordinates (elements) and the output window.
struct Tile {
  int a_mn0, a_k0;        // A: first M row (K-major) / M column (MN-major), first K element
  int b_mn0, b_k0;        // B: likewise for N
  int k_blocks;           // stages of K to accumulate (0 -> the tile is zero)
  int row0, row_lim;      // output rows [row0, row_lim) of this tile's 128 rows are stored (row index into C)
  int col0, col_lim;      // output columns
  size_t c_base;          // element offset of C(0, 0) for this tile (grouped wgrad: the expert's matrix)
};

SM90_DEVICE void raster(int local, int m_blocks, int n_blocks, int& m_blk, int& n_blk) {
  const int per_band = GROUP_M * n_blocks;
  const int band = local / per_band;
  const int first_m = band * GROUP_M;
  const int gsize = min(m_blocks - first_m, GROUP_M);
  const int in_band = local - band * per_band;
  m_blk = first_m + in_band % gsize;
  n_blk = in_band / gsize;
}

struct Epilogue {
  void* C;
  int ldc;
  int out_dtype;          // CB_F32 / CB_F16 / CB_BF16
  int accumulate;         // D += existing C
  const float* scale_a;   // fp8 dequantisation: device fp32 scalars multiplied into the product (null = 1)
  const float* scale_b;
  // int8 (W8A8) output: C = (float(acc) * row_scale[m]) * col_scale[n] + bias[n], each step rounded once
  const float* row_scale = nullptr;   // fp32 [M] per token, or one device scalar when row_scale_step == 0
  int row_scale_step = 0;
  const float* col_scale = nullptr;   // fp32 [N] per output channel
  const void* bias = nullptr;         // [N] in bias_dtype, or null
  int bias_dtype = CB_F32;
  // split-K (W8A8): the K range of an output tile is spread over `splits` CTAs that add their int32 partials into
  // split_acc [M, N] (ld N) and count arrivals per (tile, warpgroup) in split_cnt; both are zeroed by the caller.  The
  // last warpgroup to arrive runs the epilogue on the full sum.  Null = each CTA owns the whole K range of its tiles.
  int* split_acc = nullptr;
  unsigned* split_cnt = nullptr;
  int splits = 1;
};

template <typename T> SM90_DEVICE void store_pair(T* dst, float a, float b, bool two, bool acc) {
  if (two) {
    if (acc) {
      const float2 o = to_f32x2(dst);
      a += o.x; b += o.y;
    }
    store_f32x2(dst, a, b);
  } else {
    dst[0] = from_f32<T>(a + (acc ? to_f32<T>(dst[0]) : 0.f));
  }
}

// Store this thread's part of a warpgroup's 64 x 128 accumulator (rows 64 * wg .. of the tile).
SM90_DEVICE void store_acc(const float (&acc)[64], const Tile& t, const Epilogue& e, int wg) {
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int r_base = t.row0 + wg * 64 + warp * 16 + (lane >> 2);
  const float alpha = (e.scale_a ? __ldg(e.scale_a) : 1.f) * (e.scale_b ? __ldg(e.scale_b) : 1.f);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r_base + 8 * h;
    if (row >= t.row_lim) continue;
    const size_t roff = t.c_base + (size_t)row * e.ldc;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = t.col0 + 8 * j + 2 * (lane & 3);
      if (col >= t.col_lim) continue;
      const bool two = col + 1 < t.col_lim;
      const float a = acc[4 * j + 2 * h] * alpha, b = acc[4 * j + 2 * h + 1] * alpha;
      if (e.out_dtype == CB_BF16)
        store_pair((__nv_bfloat16*)e.C + roff + col, a, b, two, e.accumulate);
      else if (e.out_dtype == CB_F32)
        store_pair((float*)e.C + roff + col, a, b, two, e.accumulate);
      else
        store_pair((__half*)e.C + roff + col, a, b, two, e.accumulate);
    }
  }
}

SM90_DEVICE void named_barrier_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

SM90_DEVICE float bias_f32(const void* bias, int dtype, int col) {
  if (dtype == CB_BF16) return __bfloat162float(static_cast<const __nv_bfloat16*>(bias)[col]);
  if (dtype == CB_F16) return __half2float(static_cast<const __half*>(bias)[col]);
  return static_cast<const float*>(bias)[col];
}

// W8A8 epilogue of one element: the int32 sum converted, scaled per row then per column, biased; explicit roundings so
// that --use_fast_math contracts nothing (the result is bitwise that of the unfused PyTorch ops).
SM90_DEVICE float w8a8_value(int acc, const Epilogue& e, int row, int col) {
  float v = __fmul_rn(__int2float_rn(acc), __ldg(e.row_scale + (size_t)row * e.row_scale_step));
  v = __fmul_rn(v, __ldg(e.col_scale + col));
  return e.bias ? __fadd_rn(v, bias_f32(e.bias, e.bias_dtype, col)) : v;
}

// Store this thread's part of a warpgroup's 64 x 128 int32 accumulator through the W8A8 epilogue.  `flag` is a shared
// int of this warpgroup (split-K: tells its threads whether this CTA arrived last).
SM90_DEVICE void store_acc_w8a8(int (&acc)[64], const Tile& t, const Epilogue& e, int wg, int* flag) {
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int r_base = t.row0 + wg * 64 + warp * 16 + (lane >> 2);
  const int N = t.col_lim;
  if (e.split_acc) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_base + 8 * h;
      if (row >= t.row_lim) continue;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = t.col0 + 8 * j + 2 * (lane & 3);
        int* dst = e.split_acc + (size_t)row * N + col;
        if (col < N) atomicAdd(dst, acc[4 * j + 2 * h]);
        if (col + 1 < N) atomicAdd(dst + 1, acc[4 * j + 2 * h + 1]);
      }
    }
    __threadfence();
    named_barrier_sync(1 + wg, 128);
    if ((threadIdx.x & 127) == 0) {
      const int tile = (t.row0 / BM) * ((N + BN - 1) / BN) + t.col0 / BN;
      *flag = atomicAdd(e.split_cnt + 2 * tile + wg, 1u) == (unsigned)(e.splits - 1);
    }
    named_barrier_sync(1 + wg, 128);
    if (!*flag) return;
    __threadfence();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_base + 8 * h;
      if (row >= t.row_lim) continue;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = t.col0 + 8 * j + 2 * (lane & 3);
        const int* src = e.split_acc + (size_t)row * N + col;
        if (col < N) acc[4 * j + 2 * h] = __ldcg(src);
        if (col + 1 < N) acc[4 * j + 2 * h + 1] = __ldcg(src + 1);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r_base + 8 * h;
    if (row >= t.row_lim) continue;
    const size_t roff = (size_t)row * e.ldc;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = t.col0 + 8 * j + 2 * (lane & 3);
      if (col >= N) continue;
      const bool two = col + 1 < N;
      const float a = w8a8_value(acc[4 * j + 2 * h], e, row, col);
      const float b = two ? w8a8_value(acc[4 * j + 2 * h + 1], e, row, col + 1) : 0.f;
      if (e.out_dtype == CB_BF16)
        store_pair((__nv_bfloat16*)e.C + roff + col, a, b, two, false);
      else if (e.out_dtype == CB_F32)
        store_pair((float*)e.C + roff + col, a, b, two, false);
      else
        store_pair((__half*)e.C + roff + col, a, b, two, false);
    }
  }
}

// The wgmmas of one stage for one consumer warpgroup (rows 64 * wg of A).
template <int KIND, int A_MN, int B_MN, typename Acc>
SM90_DEVICE void mma_stage(Acc (&acc)[64], uint32_t sa, uint32_t sb, int wg) {
  using KT = KindTraits<KIND>;
  // A: K-major rows 64 wg .. 64 wg + 63 start 64 rows x 128 B = 8 KB in; MN-major column chunk wg is 8 KB in as well
  const uint64_t da = make_smem_desc_sw128(sa + wg * 8192, A_MN ? 8192 : 16, 1024);
  const uint64_t db = make_smem_desc_sw128(sb, B_MN ? 8192 : 16, 1024);
#pragma unroll
  for (int k = 0; k < KT::KE / KT::MMA_K; ++k) {
    const uint32_t ao = A_MN ? k * 2048 : k * 32;
    const uint32_t bo = B_MN ? k * 2048 : k * 32;
    const uint64_t a = advance_desc(da, ao), b = advance_desc(db, bo);
    if constexpr (KIND == K_BF16) wgmma_ss_m64n128k16_bf16<A_MN, B_MN>(acc, a, b);
    else if constexpr (KIND == K_F16) wgmma_ss_m64n128k16_f16<A_MN, B_MN>(acc, a, b);
    else if constexpr (KIND == K_E4M3_E4M3) wgmma_ss_m64n128k32_e4m3_e4m3(acc, a, b);
    else if constexpr (KIND == K_E4M3_E5M2) wgmma_ss_m64n128k32_e4m3_e5m2(acc, a, b);
    else if constexpr (KIND == K_E5M2_E4M3) wgmma_ss_m64n128k32_e5m2_e4m3(acc, a, b);
    else if constexpr (KIND == K_E5M2_E5M2) wgmma_ss_m64n128k32_e5m2_e5m2(acc, a, b);
    else wgmma_ss_m64n128k32_s8_s8(acc, a, b);
  }
}

struct Smem {
  uint8_t* a;
  uint8_t* b;
  uint64_t* full;
  uint64_t* empty;
};

SM90_DEVICE Smem carve(uint8_t* smem_raw) {
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  Smem s;
  s.a = smem;
  s.b = smem + STAGES * A_BYTES;
  s.full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  s.empty = s.full + STAGES;
  return s;
}

// thread 0 of the CTA; the caller synchronises the CTA afterwards
SM90_DEVICE void init_barriers(const Smem& s) {
  for (int i = 0; i < STAGES; ++i) {
    mbar_init(&s.full[i], 1);
    mbar_init(&s.empty[i], 2);   // one arrival per consumer warpgroup
  }
  fence_barrier_init();
}

// Producer warp: TMA loads of every tile this CTA owns.
template <int KIND, int A_MN, int B_MN, class Prob>
SM90_DEVICE void producer(const CUtensorMap* ta, const CUtensorMap* tb, const Prob& prob, const Smem& s, int num_tiles) {
  using KT = KindTraits<KIND>;
  const int lane = threadIdx.x & 31;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const Tile t = prob.tile(tile);
    if (lane == 0) prob.before_load(tile, t);
    __syncwarp();
    for (int kb = 0; kb < t.k_blocks; ++kb) {
      mbar_wait(&s.empty[stage], phase ^ 1);
      if (lane == 0) {
        mbar_arrive_expect_tx(&s.full[stage], STAGE_BYTES);
        uint8_t* sa = s.a + stage * A_BYTES;
        uint8_t* sb = s.b + stage * B_BYTES;
        const int ka = t.a_k0 + kb * KT::KE, kbb = t.b_k0 + kb * KT::KE;
        if (!A_MN) {
          tma_load_2d(ta, &s.full[stage], sa, ka, t.a_mn0);                         // box [128 rows, 128 B]
        } else {
#pragma unroll
          for (int j = 0; j < 2; ++j) tma_load_2d(ta, &s.full[stage], sa + j * 8192, t.a_mn0 + j * 64, ka);   // [64 k, 64]
        }
        if (!B_MN) {
          tma_load_2d(tb, &s.full[stage], sb, kbb, t.b_mn0);
        } else {
#pragma unroll
          for (int j = 0; j < 2; ++j) tma_load_2d(tb, &s.full[stage], sb + j * 8192, t.b_mn0 + j * 64, kbb);
        }
      }
      __syncwarp();
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
  }
}

// Consumer warpgroups: main loop + epilogue of every tile this CTA owns.
template <int KIND, int A_MN, int B_MN, class Prob>
SM90_DEVICE void consumer(const Prob& prob, const Smem& s, const Epilogue& e, int num_tiles) {
  const int wg = threadIdx.x >> 7;
  const bool leader = (threadIdx.x & 127) == 0;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const Tile t = prob.tile(tile);
    typename KindTraits<KIND>::Acc acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0;
    int prev = -1;
    for (int kb = 0; kb < t.k_blocks; ++kb) {
      mbar_wait(&s.full[stage], phase);
      if constexpr (KindTraits<KIND>::F8) {
        // the fp8 tensor-core accumulator keeps fewer mantissa bits than fp32: every stage (128 K) is summed in a
        // fresh partial and promoted into the fp32 accumulator
        float part[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) part[i] = 0.f;
        wgmma_fence();
        mma_stage<KIND, A_MN, B_MN>(part, smem_u32(s.a + stage * A_BYTES), smem_u32(s.b + stage * B_BYTES), wg);
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(part);
        if (leader) mbar_arrive(&s.empty[stage]);
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] += part[i];
      } else {
        wgmma_fence();
        mma_stage<KIND, A_MN, B_MN>(acc, smem_u32(s.a + stage * A_BYTES), smem_u32(s.b + stage * B_BYTES), wg);
        wgmma_commit();
        wgmma_wait<1>();                                 // the group of the previous stage has retired
        if (prev >= 0 && leader) mbar_arrive(&s.empty[prev]);
        prev = stage;
      }
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (prev >= 0 && leader) mbar_arrive(&s.empty[prev]);
    if constexpr (KindTraits<KIND>::S8)
      store_acc_w8a8(acc, t, e, wg, reinterpret_cast<int*>(s.empty + STAGES) + wg);
    else
      store_acc(acc, t, e, wg);
    prob.after_store(tile, t, wg);
  }
}

// Plain problem: C[M, N] over K, tiles rasterised in bands of GROUP_M row blocks (L2 reuse of B).
struct DenseProb {
  int M, N, K, ke;        // ke: K elements per stage
  int m_blocks, n_blocks;
  SM90_DEVICE int num_tiles() const { return m_blocks * n_blocks; }
  SM90_DEVICE Tile tile(int idx) const {
    int mb, nb;
    raster(idx, m_blocks, n_blocks, mb, nb);
    Tile t;
    t.a_mn0 = mb * BM; t.a_k0 = 0;
    t.b_mn0 = nb * BN; t.b_k0 = 0;
    t.k_blocks = (K + ke - 1) / ke;
    t.row0 = mb * BM; t.row_lim = M;
    t.col0 = nb * BN; t.col_lim = N;
    t.c_base = 0;
    return t;
  }
  SM90_DEVICE void before_load(int, const Tile&) const {}
  SM90_DEVICE void after_store(int, const Tile&, int) const {}
};

template <int KIND, int A_MN, int B_MN, class Prob>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const Prob prob,
            const Epilogue e) {
  extern __shared__ uint8_t smem_raw[];
  const Smem s = carve(smem_raw);
  const int num_tiles = prob.num_tiles();
  if (threadIdx.x == 0) init_barriers(s);
  if (threadIdx.x == CONSUMER_THREADS) {
    prefetch_tensormap(&tmap_a);
    prefetch_tensormap(&tmap_b);
  }
  __syncthreads();
  if ((int)(threadIdx.x >> 5) == PRODUCER_WARP)
    producer<KIND, A_MN, B_MN>(&tmap_a, &tmap_b, prob, s, num_tiles);
  else
    consumer<KIND, A_MN, B_MN>(prob, s, e, num_tiles);
}

// Host: opt in to the shared memory once per instantiation and launch.
template <int KIND, int A_MN, int B_MN, class Prob>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const Prob& prob, const Epilogue& e, int grid,
           cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t err = cudaFuncSetAttribute(gemm_kernel<KIND, A_MN, B_MN, Prob>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (err != cudaSuccess) return (int)err;
    attr_set = true;
  }
  if (grid <= 0) return 0;
  gemm_kernel<KIND, A_MN, B_MN, Prob><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(ta, tb, prob, e);
  return (int)cudaGetLastError();
}

// Host: can store_acc write this output?  out_dtype must be one it knows (any other code would be stored as fp16), and
// since two adjacent columns go out as one 2-element store (float2 / __nv_bfloat162 / __half2), C's base must be
// aligned to two elements and ldc must be even (and at least the row width n).
inline bool epilogue_ok(const void* C, long long ldc, long long n, int out_dtype) {
  if (out_dtype != CB_F32 && out_dtype != CB_F16 && out_dtype != CB_BF16) return false;
  const uintptr_t pair_bytes = out_dtype == CB_F32 ? 8 : 4;
  return ldc >= n && (ldc & 1) == 0 && reinterpret_cast<uintptr_t>(C) % pair_bytes == 0;
}

// Runtime (a_mn, b_mn, kind) -> template instantiation for 16-bit operands.
template <class Prob>
int launch16(const CUtensorMap& ta, const CUtensorMap& tb, const Prob& prob, const Epilogue& e, int grid, bool bf16,
             int a_mn, int b_mn, cudaStream_t st) {
#define CB_L(K, A, B) return launch<K, A, B>(ta, tb, prob, e, grid, st)
  if (bf16) {
    if (!a_mn && !b_mn) CB_L(K_BF16, 0, 0);
    if (!a_mn && b_mn) CB_L(K_BF16, 0, 1);
    if (a_mn && !b_mn) CB_L(K_BF16, 1, 0);
    CB_L(K_BF16, 1, 1);
  }
  if (!a_mn && !b_mn) CB_L(K_F16, 0, 0);
  if (!a_mn && b_mn) CB_L(K_F16, 0, 1);
  if (a_mn && !b_mn) CB_L(K_F16, 1, 0);
  CB_L(K_F16, 1, 1);
#undef CB_L
}

// Tensor maps of the two operands.  K-major operand: tensor [rows = M/N, cols = K], box [128, 128 B].  MN-major:
// tensor [rows = K, cols = M/N], box [64 K rows, 64].
inline int tmap16(CUtensorMap* m, const void* p, bool mn_major, uint64_t mn, uint64_t k, uint64_t ld, bool bf16) {
  return mn_major ? make_tmap_2d_16b(m, p, k, mn, ld, 64, 64, bf16) : make_tmap_2d_16b(m, p, mn, k, ld, 128, 64, bf16);
}

}  // namespace gemm90
