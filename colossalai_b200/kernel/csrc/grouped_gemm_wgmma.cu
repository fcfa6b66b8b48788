// Grouped (per-expert) wgmma GEMM for sm_90a: the three GEMMs of a mixture-of-experts MLP over token rows that are
// grouped by expert, with the group boundaries read ON THE DEVICE (no host sync, no per-expert launches).
//
//   MODE_NT  (forward)  Y[rows of e, N]  = X[rows of e, K] x W[e][N, K]^T         variable M per group
//   MODE_NN  (dgrad)    dX[rows of e, N] = dY[rows of e, K] x W[e][K, N]           variable M per group
//   MODE_TN  (wgrad)    dW[e][M, N]     (+)= dY[rows of e, M]^T x X[rows of e, N]  variable K (= rows) per group
//
// `offs[e]` is the exclusive end row of group e (cumulative counts, int32, device memory).  One persistent launch of
// the 128 x 128 wgmma main loop of gemm_sm90.cuh; every role walks the same tile list, which is built from `offs` at
// kernel start:
//   * variable-M modes: group e contributes ceil(rows_e / 128) row tiles x ceil(N / 128) column tiles, rasterised inside
//     the group in bands of 8 row tiles (L2 reuse of the expert's weight tile).  A row tile that runs past the end of its
//     group simply loads rows of the next group (or TMA zero fill) and masks them at the store - no padding needed;
//   * variable-K mode: every group owns (M / 128) x (N / 128) tiles whose reduction runs over the group's token rows; the
//     row range of a group must start and end on a multiple of 128 - the dispatch lays groups out that way
//     (`moe/grouped_gemm.py` pads with zero rows otherwise) - so a k-block never mixes two experts.
//
// Replaces the reference's python loop over local experts (`shardformer/modeling/mixtral.py:177-191`) and round 1's
// library `torch._grouped_mm`.
#include "gemm_sm90.cuh"

using namespace gemm90;

namespace {

constexpr int MAX_GROUPS = 512;
constexpr int KE = 64;                 // K elements per stage (16-bit operands)
constexpr int SMEM_TOTAL = SMEM_BYTES + (MAX_GROUPS + 1) * 4;

enum { MODE_NT = 0, MODE_NN = 1, MODE_TN = 2 };

struct GroupedParams {
  const int* offs;          // [E] cumulative row ends
  int E;
  int total_rows;           // rows of the grouped operand(s) (buffer size; >= offs[E-1])
  int M, N, K;              // NT / NN: N = output columns, K = reduction; TN: M x N = per-expert output, K unused
  long long c_group_stride; // TN: elements between the outputs of consecutive experts
  int b_group_rows;         // NT: N rows per expert in the [E * N, K] view of W; NN: K rows per expert in [E * K, N]
};

template <int MODE> struct GroupedProb {
  GroupedParams p;
  const int* tile_start;    // shared memory, [E + 1]: row tiles of the groups before e (variable-M modes)
  int n_blocks;
  int num;
  SM90_DEVICE int num_tiles() const { return num; }
  SM90_DEVICE Tile tile(int idx) const {
    Tile t;
    if (MODE == MODE_TN) {
      const int m_blocks = (p.M + BM - 1) / BM;
      const int per_group = m_blocks * n_blocks;
      const int g = idx / per_group;
      int mb, nb;
      raster(idx - g * per_group, m_blocks, n_blocks, mb, nb);
      const int r0 = g == 0 ? 0 : p.offs[g - 1];
      const int r1 = p.offs[g];
      t.a_mn0 = mb * BM; t.a_k0 = r0;
      t.b_mn0 = nb * BN; t.b_k0 = r0;
      t.k_blocks = r1 > r0 ? (r1 - r0 + KE - 1) / KE : 0;    // an expert without tokens: its gradient is zero
      t.row0 = mb * BM; t.row_lim = p.M;
      t.col0 = nb * BN; t.col_lim = p.N;
      t.c_base = (size_t)g * (size_t)p.c_group_stride;
      return t;
    }
    // group of this tile: last e with tile_start[e] * n_blocks <= idx
    int lo = 0, hi = p.E - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tile_start[mid] * n_blocks <= idx) lo = mid; else hi = mid - 1;
    }
    const int g = lo;
    int mb, nb;
    raster(idx - tile_start[g] * n_blocks, tile_start[g + 1] - tile_start[g], n_blocks, mb, nb);
    const int g0 = g == 0 ? 0 : p.offs[g - 1];
    t.a_mn0 = g0 + mb * BM; t.a_k0 = 0;
    if (MODE == MODE_NT) { t.b_mn0 = g * p.b_group_rows + nb * BN; t.b_k0 = 0; }        // W as [E * N, K]
    else { t.b_mn0 = nb * BN; t.b_k0 = g * p.b_group_rows; }                             // W as [E * K, N]
    t.k_blocks = (p.K + KE - 1) / KE;
    t.row0 = g0 + mb * BM; t.row_lim = p.offs[g];
    t.col0 = nb * BN; t.col_lim = p.N;
    t.c_base = 0;
    return t;
  }
  SM90_DEVICE void before_load(int, const Tile&) const {}
  SM90_DEVICE void after_store(int, const Tile&, int) const {}
};

template <int MODE, int KIND>
__global__ void __launch_bounds__(NUM_THREADS, 1)
grouped_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                    const GroupedParams p, const Epilogue e) {
  constexpr int A_MN = MODE == MODE_TN;
  constexpr int B_MN = MODE != MODE_NT;
  extern __shared__ uint8_t smem_raw[];
  const Smem s = carve(smem_raw);
  int* tile_start = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(s.full) + 256);
  GroupedProb<MODE> prob;
  prob.p = p;
  prob.tile_start = tile_start;
  prob.n_blocks = (p.N + BN - 1) / BN;
  if (threadIdx.x == 0) {
    init_barriers(s);
    if (MODE != MODE_TN) {
      int acc = 0, prev = 0;
      for (int g = 0; g < p.E; ++g) {
        tile_start[g] = acc;
        const int end = p.offs[g];
        acc += (end - prev + BM - 1) / BM;
        prev = end;
      }
      tile_start[p.E] = acc;
    }
  }
  if (threadIdx.x == CONSUMER_THREADS) {
    prefetch_tensormap(&tmap_a);
    prefetch_tensormap(&tmap_b);
  }
  __syncthreads();
  prob.num = MODE == MODE_TN ? p.E * ((p.M + BM - 1) / BM) * prob.n_blocks : tile_start[p.E] * prob.n_blocks;
  if ((int)(threadIdx.x >> 5) == PRODUCER_WARP)
    producer<KIND, A_MN, B_MN>(&tmap_a, &tmap_b, prob, s, prob.num);
  else
    consumer<KIND, A_MN, B_MN>(prob, s, e, prob.num);
}

template <int MODE, int KIND>
int launch_grouped_k(const CUtensorMap& ta, const CUtensorMap& tb, const GroupedParams& p, const Epilogue& e,
                     cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t err = cudaFuncSetAttribute(grouped_gemm_kernel<MODE, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SMEM_TOTAL);
    if (err != cudaSuccess) return (int)err;
    attr_set = true;
  }
  // the number of tiles is only known on the device: full persistent grid
  grouped_gemm_kernel<MODE, KIND><<<cb_num_sms(), NUM_THREADS, SMEM_TOTAL, stream>>>(ta, tb, p, e);
  return (int)cudaGetLastError();
}

template <int MODE>
int launch_grouped(const CUtensorMap& ta, const CUtensorMap& tb, const GroupedParams& p, const Epilogue& e, bool bf16,
                   cudaStream_t stream) {
  return bf16 ? launch_grouped_k<MODE, K_BF16>(ta, tb, p, e, stream) : launch_grouped_k<MODE, K_F16>(ta, tb, p, e, stream);
}

}  // namespace

extern "C" {

// Variable-M grouped GEMM.  x [total_rows, K] (rows grouped by expert, `offs` = cumulative row ends on the device);
// transpose_b != 0: w [E, N, K] and y = x w[e]^T (forward);  transpose_b == 0: w [E, K, N] and y = x w[e] (dgrad with
// the forward weight [E, K(out), N(in)]).  y [total_rows, N].  Requirements: contiguous w, K % 8 == 0, K >= 8,
// N % 8 == 0, 16-byte aligned x / w, y aligned to 4 bytes with ldy even and >= N, E <= 512; transpose_b == 0
// additionally needs K % 128 == 0 (a k-block must not straddle two experts' weights).  Rows after offs[E - 1] are
// neither read into any group nor written.
int cb_grouped_gemm(const void* x, const void* w, void* y, const int* offs, int E, int total_rows, int N, int K, int ldx,
                    int ldy, int transpose_b, int dtype, cudaStream_t stream) {
  if (E > MAX_GROUPS || (dtype != CB_BF16 && dtype != CB_F16) || K <= 0 || (K & 7) || (N & 7) ||
      !epilogue_ok(y, ldy, N, dtype))
    return (int)cudaErrorInvalidValue;
  if (!transpose_b && (K % 128)) return (int)cudaErrorInvalidValue;
  if (E <= 0 || total_rows <= 0 || N <= 0) return 0;
  const bool bf16 = dtype == CB_BF16;
  CUtensorMap ta, tb;
  int r = tmap16(&ta, x, false, total_rows, K, ldx, bf16);
  if (r) return 1000 + r;
  GroupedParams p{};
  p.offs = offs; p.E = E; p.total_rows = total_rows; p.N = N; p.K = K;
  const Epilogue e{y, ldy, dtype, 0, nullptr, nullptr};
  if (transpose_b) {
    r = tmap16(&tb, w, false, (uint64_t)E * N, K, K, bf16);
    if (r) return 2000 + r;
    p.b_group_rows = N;
    return launch_grouped<MODE_NT>(ta, tb, p, e, bf16, stream);
  }
  r = tmap16(&tb, w, true, N, (uint64_t)E * K, N, bf16);
  if (r) return 2000 + r;
  p.b_group_rows = K;
  return launch_grouped<MODE_NN>(ta, tb, p, e, bf16, stream);
}

// Variable-K grouped GEMM (weight gradients): dw[e] [M, N] (+)= dy[rows of e, M]^T x[rows of e, N].  Every group's row
// range must start and end on a multiple of 128.  out_dtype: bf16 / fp16 / fp32, dw [E, M, N] contiguous and aligned to
// two output elements, total_rows >= 1 (the operands' tensor maps cannot be empty).  An expert without rows gets
// dw[e] = 0 (or keeps dw[e] when accumulating).
int cb_grouped_gemm_wgrad(const void* dy, const void* x, void* dw, const int* offs, int E, int total_rows, int M, int N,
                          int lddy, int ldx, int in_dtype, int out_dtype, int accumulate, cudaStream_t stream) {
  if (E > MAX_GROUPS || (in_dtype != CB_BF16 && in_dtype != CB_F16) || (M & 7) || (N & 7) || total_rows <= 0 ||
      !epilogue_ok(dw, N, N, out_dtype))
    return (int)cudaErrorInvalidValue;
  if (E <= 0 || M <= 0 || N <= 0) return 0;
  const bool bf16 = in_dtype == CB_BF16;
  CUtensorMap ta, tb;
  int r = tmap16(&ta, dy, true, M, total_rows, lddy, bf16);
  if (r) return 1000 + r;
  r = tmap16(&tb, x, true, N, total_rows, ldx, bf16);
  if (r) return 2000 + r;
  GroupedParams p{};
  p.offs = offs; p.E = E; p.total_rows = total_rows; p.M = M; p.N = N; p.K = 0;
  p.c_group_stride = (long long)M * N;
  const Epilogue e{dw, N, out_dtype, accumulate, nullptr, nullptr};
  return launch_grouped<MODE_TN>(ta, tb, p, e, bf16, stream);
}

}  // extern "C"
