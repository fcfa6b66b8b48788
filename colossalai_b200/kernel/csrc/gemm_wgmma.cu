// Dense GEMMs for sm_90a on the wgmma main loop of gemm_sm90.cuh:
//
//   D[M,N] (+)= sum_k A(m,k) * B(n,k),  bf16/fp16 in, fp32 accumulate in registers, bf16/fp16/fp32 out, where A and B
//   may each be K-major or MN-major - the three GEMMs of a linear layer without any transposition pass:
//       fwd   y  = x  W^T : A = x  (K-major),  B = W  (K-major)
//       dgrad dx = dy W   : A = dy (K-major),  B = W  (MN-major: stored [N_out(red), K_in])
//       wgrad dW = dy^T x : A = dy (MN-major), B = x  (MN-major), optional fp32/bf16 accumulation into main_grad;
//   and the 8-bit float variant (E4M3 / E5M2, both operands K-major) with per-tensor dequantisation scales.
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

int cb_gemm_smem_bytes(int block_n) {
  (void)block_n;
  return SMEM_BYTES;
}

}  // extern "C"
