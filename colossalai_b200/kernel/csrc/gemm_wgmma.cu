// Dense GEMMs for sm_90a on the wgmma main loop of gemm_sm90.cuh:
//
//   D[M,N] (+)= sum_k A(m,k) * B(n,k),  bf16/fp16 in, fp32 accumulate in registers, bf16/fp16/fp32 out, where A and B
//   may each be K-major or MN-major - the three GEMMs of a linear layer without any transposition pass:
//       fwd   y  = x  W^T : A = x  (K-major),  B = W  (K-major)
//       dgrad dx = dy W   : A = dy (K-major),  B = W  (MN-major: stored [N_out(red), K_in])
//       wgrad dW = dy^T x : A = dy (MN-major), B = x  (MN-major), optional fp32/bf16 accumulation into main_grad;
//   and the 8-bit float variant (E4M3 / E5M2, both operands K-major) with per-tensor dequantisation scales;
//   and the int8 W8A8 variant (s8 x s8 -> exact int32) with the SmoothQuant epilogue (per-token x per-channel scales,
//   bias), split over K for small-M (decode) shapes.
//
// Grid = min(#tiles, #SMs) persistent CTAs of 128 x 128 tiles.
//
// This kernel replaces the reference's cuBLAS calls (`F.linear` / `torch.matmul` in shardformer/layer/_operation.py)
// with our own tensor-core path; the comm-fused variants in fused_comm_gemm.cu share its main loop.
#include "gemm_sm90.cuh"

using namespace gemm90;

namespace {

DenseProb dense(int M, int N, int K, int ke) {
  DenseProb p;
  p.M = M; p.N = N; p.K = K; p.ke = ke;
  p.m_blocks = (M + BM - 1) / BM;
  p.n_blocks = (N + BN - 1) / BN;
  return p;
}

int grid_for(const DenseProb& p) {
  const int tiles = p.m_blocks * p.n_blocks;
  return tiles < cb_num_sms() ? tiles : cb_num_sms();
}

// |acc| <= 127 * 127 * K must fit in int32
constexpr int W8A8_MAX_K = 133143;

// Dense W8A8 problem with the K range of every output tile split over `splits` consecutive work items (kbs stages each).
struct SplitKProb {
  int M, N, K, splits, kbs;
  int m_blocks, n_blocks;
  SM90_DEVICE int num_tiles() const { return m_blocks * n_blocks * splits; }
  SM90_DEVICE Tile tile(int idx) const {
    int mb, nb;
    raster(idx / splits, m_blocks, n_blocks, mb, nb);
    const int k0 = (idx % splits) * kbs * 128;
    Tile t;
    t.a_mn0 = mb * BM; t.a_k0 = k0;
    t.b_mn0 = nb * BN; t.b_k0 = k0;
    t.k_blocks = min(kbs, (K - k0 + 127) / 128);
    t.row0 = mb * BM; t.row_lim = M;
    t.col0 = nb * BN; t.col_lim = N;
    t.c_base = 0;
    return t;
  }
  SM90_DEVICE void before_load(int, const Tile&) const {}
  SM90_DEVICE void after_store(int, const Tile&, int) const {}
};

// Split-K for shapes whose tiles fill at most half the SMs (decode: M <= 64 gives N / 128 tiles) and whose K is long
// next to M (K >= 128 M: the int32 partials each split adds grow with M, the wait for one CTA's serial K loop with K):
// as many splits as fit on the SMs, each at least 4 stages (512) of K deep.  Measured on an H100 (docs/kernels.md),
// splitting was 1.1-1.5x faster for the Llama-3-8B down projection (K 14336) at M <= 64 and about even at K 4096,
// M <= 16, but up to 1.7x slower at K 4096, M 64-256.  Returns the problem; splits == 1 means no split.
SplitKProb w8a8_problem(int M, int N, int K) {
  SplitKProb p;
  p.M = M; p.N = N; p.K = K;
  p.m_blocks = (M + BM - 1) / BM;
  p.n_blocks = (N + BN - 1) / BN;
  const int tiles = p.m_blocks * p.n_blocks, kblocks = (K + 127) / 128, sms = cb_num_sms();
  int splits = 2 * tiles <= sms && K >= 128LL * M ? min(sms / tiles, kblocks / 4) : 1;
  if (splits < 2) splits = 1;
  p.kbs = (kblocks + splits - 1) / splits;
  p.splits = (kblocks + p.kbs - 1) / p.kbs;   // no empty split
  return p;
}

long long w8a8_workspace_bytes(const SplitKProb& p) {
  return p.splits > 1 ? 4LL * ((long long)p.M * p.N + 2LL * p.m_blocks * p.n_blocks) : 0;
}

}  // namespace

extern "C" {

// D[M,N] (+)= A x B^T-like contraction over K.
//   a_mn_major == 0: A is [M, K] row-major with leading dimension lda;  == 1: A is stored [K, M] (lda between K rows)
//   b_mn_major == 0: B is [N, K] row-major with leading dimension ldb;  == 1: B is stored [K, N]
// Requirements: 16-byte aligned A / B bases, lda / ldb multiples of 8 elements, K >= 1; out_dtype fp32 / fp16 / bf16,
// C aligned to two output elements, ldc even and >= N.  M, N, K are otherwise arbitrary (TMA zero-fills out-of-bounds,
// stores are predicated).  Anything else returns cudaErrorInvalidValue before any work.  `block_n` is accepted for
// interface stability; the tile is always 128 x 128.
int cb_gemm_tcgen05(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                    int a_mn_major, int b_mn_major, int in_dtype, int out_dtype, int accumulate, int block_n,
                    cudaStream_t stream) {
  (void)block_n;
  if (in_dtype != CB_BF16 && in_dtype != CB_F16) return (int)cudaErrorInvalidValue;
  // K == 0 would need tensor maps of an empty operand, which the driver refuses
  if (K <= 0 || !epilogue_ok(C, ldc, N, out_dtype)) return (int)cudaErrorInvalidValue;
  if (M <= 0 || N <= 0) return 0;
  const bool bf16 = in_dtype == CB_BF16;
  CUtensorMap ta, tb;
  int r = tmap16(&ta, A, a_mn_major, M, K, lda, bf16);
  if (r) return 1000 + r;
  r = tmap16(&tb, B, b_mn_major, N, K, ldb, bf16);
  if (r) return 2000 + r;
  const DenseProb p = dense(M, N, K, 64);
  const Epilogue e{C, ldc, out_dtype, accumulate, nullptr, nullptr};
  return launch16(ta, tb, p, e, grid_for(p), bf16, a_mn_major, b_mn_major, stream);
}

// D[M,N] (+)= scale_a * scale_b * (A[M,K] x B[N,K]^T) with 8-bit float operands (wgmma m64n128k32, 128 K-elements per
// stage).  a_fmt / b_fmt: 0 = E4M3, 1 = E5M2.  Requirements: 16-byte aligned bases, lda / ldb multiples of 16 bytes,
// K >= 1, and the output rules of cb_gemm_tcgen05.  scale pointers are device fp32 scalars or null.  With accumulate,
// D = scale_a * scale_b * (A x B^T) + C: the scales apply to the product only.
int cb_gemm_fp8_tcgen05(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                        int a_fmt, int b_fmt, int out_dtype, int accumulate, const float* scale_a,
                        const float* scale_b, cudaStream_t stream) {
  if ((lda & 15) || (ldb & 15) || K <= 0 || !epilogue_ok(C, ldc, N, out_dtype)) return (int)cudaErrorInvalidValue;
  if (M <= 0 || N <= 0) return 0;
  CUtensorMap ta, tb;
  int r = make_tmap_2d_8b(&ta, A, M, K, lda, 128, 128);
  if (r) return 1000 + r;
  r = make_tmap_2d_8b(&tb, B, N, K, ldb, 128, 128);
  if (r) return 2000 + r;
  const DenseProb p = dense(M, N, K, 128);
  const Epilogue e{C, ldc, out_dtype, accumulate, scale_a, scale_b};
  const int g = grid_for(p);
  const int kind = 2 + (a_fmt & 1) * 2 + (b_fmt & 1);
  if (kind == K_E4M3_E4M3) return launch<K_E4M3_E4M3, 0, 0>(ta, tb, p, e, g, stream);
  if (kind == K_E4M3_E5M2) return launch<K_E4M3_E5M2, 0, 0>(ta, tb, p, e, g, stream);
  if (kind == K_E5M2_E4M3) return launch<K_E5M2_E4M3, 0, 0>(ta, tb, p, e, g, stream);
  return launch<K_E5M2_E5M2, 0, 0>(ta, tb, p, e, g, stream);
}

// W8A8: C[M,N] = (float(A x B^T) * row_scale[m]) * col_scale[n] (+ bias[n]), A int8 [M, K], B int8 [N, K] (both
// row-major), exact int32 accumulation, one rounding to the output dtype.  row_scale: fp32 [M] (row_scale_per_row = 1,
// per-token activation scales) or one device fp32 scalar (0, static); col_scale: fp32 [N]; bias: null or [N] of
// bias_dtype (fp32 / fp16 / bf16).  Requirements: 16-byte aligned A / B bases, lda / ldb multiples of 16 bytes and
// >= K, 1 <= K <= 133143 (int32 range of the sum), non-null scales, and the output rules of cb_gemm_tcgen05.  Shapes
// with few output tiles split K across CTAs: they need `workspace` zeroed on `stream`, of at least
// cb_gemm_w8a8_workspace(M, N, K) bytes (0 = no split, workspace may be null).  Anything else returns
// cudaErrorInvalidValue before any work.
int cb_gemm_w8a8(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                 const float* row_scale, int row_scale_per_row, const float* col_scale, const void* bias,
                 int bias_dtype, int out_dtype, void* workspace, long long workspace_bytes, cudaStream_t stream) {
  if (reinterpret_cast<uintptr_t>(A) % 16 || reinterpret_cast<uintptr_t>(B) % 16 || (lda & 15) || (ldb & 15) ||
      lda < K || ldb < K || K <= 0 || K > W8A8_MAX_K || !row_scale || !col_scale ||
      (bias && bias_dtype != CB_F32 && bias_dtype != CB_F16 && bias_dtype != CB_BF16) ||
      !epilogue_ok(C, ldc, N, out_dtype))
    return (int)cudaErrorInvalidValue;
  if (M <= 0 || N <= 0) return 0;
  const SplitKProb p = w8a8_problem(M, N, K);
  const long long need = w8a8_workspace_bytes(p);
  if (need && (!workspace || workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 4))
    return (int)cudaErrorInvalidValue;
  CUtensorMap ta, tb;
  int r = make_tmap_2d_8b(&ta, A, M, K, lda, 128, 128);
  if (r) return 1000 + r;
  r = make_tmap_2d_8b(&tb, B, N, K, ldb, 128, 128);
  if (r) return 2000 + r;
  Epilogue e{C, ldc, out_dtype, 0, nullptr, nullptr};
  e.row_scale = row_scale;
  e.row_scale_step = row_scale_per_row ? 1 : 0;
  e.col_scale = col_scale;
  e.bias = bias;
  e.bias_dtype = bias_dtype;
  if (need) {
    e.split_acc = static_cast<int*>(workspace);
    e.split_cnt = reinterpret_cast<unsigned*>(e.split_acc + (size_t)M * N);
    e.splits = p.splits;
  }
  const int work = p.m_blocks * p.n_blocks * p.splits;
  return launch<K_S8, 0, 0>(ta, tb, p, e, work < cb_num_sms() ? work : cb_num_sms(), stream);
}

// Bytes of zeroed workspace cb_gemm_w8a8 needs for this shape (0: the shape runs without split-K).
long long cb_gemm_w8a8_workspace(int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  return w8a8_workspace_bytes(w8a8_problem(M, N, K));
}

int cb_gemm_smem_bytes(int block_n) {
  (void)block_n;
  return SMEM_BYTES;
}

}  // extern "C"
