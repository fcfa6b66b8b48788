// Flash attention forward and backward for sm_90a on warpgroup MMA (wgmma).
//
//   O = softmax(scale * Q K^T + mask) V,   LSE = log sum exp     (GQA: Hq = g * Hkv, head_dim 64 or 128)
//
// FORWARD.  One CTA = one 128-row query tile of one (batch, head); 288 threads:
//   warps 0..7  two consumer warpgroups, each owning 64 query rows: S_j = Q K_j^T (wgmma, both operands in shared
//               memory, fp32 accumulator in registers), online softmax in the exp2 domain on the registers, then
//               O += P_j V_j with P_j taken straight from registers as the A operand (no shared-memory round trip) and
//               V_j read MN-major from shared memory;
//   warp 8      TMA producer: Q once, then (K_j, V_j) tiles of 128 keys through a 2-stage mbarrier ring.
// Shared memory: Q 128 x D + 2 x (K 128 x D + V 128 x D), SWIZZLE_128B, = 160 KB at D = 128.
//
// Reference being replaced: flash-attn 2 `flash_attn_func` / `_flash_attn_varlen_forward` (mma.sync kernels) used by
// `colossalai/shardformer/layer/attn.py:356-372,720-755`.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "sm90.cuh"

namespace {
using namespace sm90;

constexpr int BLOCK_Q = 128;
constexpr int BLOCK_KV = 128;
constexpr int NUM_THREADS = 288;
constexpr int PRODUCER_WARP = 8;
constexpr int KV_STAGES = 2;
constexpr float LOG2E = 1.4426950408889634f;

template <int D> struct FaCfg {
  static constexpr int Q_BYTES = BLOCK_Q * D * 2;
  static constexpr int K_BYTES = BLOCK_KV * D * 2;
  static constexpr int V_BYTES = BLOCK_KV * D * 2;
  static constexpr int KV_STAGE_BYTES = K_BYTES + V_BYTES;
  static constexpr int SMEM_BYTES = Q_BYTES + KV_STAGES * KV_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

struct FaParams {
  // packed / variable-length batches: cu_seqlens[b] .. cu_seqlens[b + 1] are the token rows of sequence b (self
  // attention, the same boundaries for queries and keys); null = `batch` equal-length sequences
  const int* cu_seqlens;
  int batch, seqlen_q, seqlen_k;     // equal-length sequences, token-major tensors [batch * seqlen, heads * D]
  int hq, hkv;
  int causal;
  float scale_log2;                  // softmax scale * log2(e)
  void* out;                         // [batch * seqlen_q, hq * D]
  float* lse;                        // [batch * seqlen_q, hq] natural-log LSE
  // ring / blockwise attention: the online-softmax state of every query row lives in (o_state, lse) between launches.
  // has_prev: start from that state (m = lse, l = 1, acc = o_state) instead of (-inf, 0, 0); the result - the merge of
  // the previous partial result with this launch's keys - is written back in fp32.  No separate rescale / merge pass.
  float* o_state;                    // [rows, hq * D] fp32, or null (plain attention: `out` in the input dtype)
  int has_prev;
  int out_dtype;
  // EXTRA variant of the kernel only (inference prefill of sliding-window / ALiBi models):
  int window;                        // > 0: query q sees keys (q - window, q]; key tiles left of every window are skipped
  const float* alibi;                // [hq] slopes (score += slope * (key - query)), or null
  // PAGED variant only (prefill over a paged KV cache): sequence b's cu_seqlens[b + 1] - cu_seqlens[b] new query rows
  // sit at the absolute positions seq_lens_k[b] - n_b .. seq_lens_k[b] - 1 and see the keys 0 .. seq_lens_k[b] - 1,
  // read from cache blocks block_tables[b][key / block_size] (k / v tensor maps over [kv_rows, hkv * D])
  const int* block_tables;           // [batch, max_blocks] int32
  const int* seq_lens_k;             // [batch] int32: cached + new tokens
  int block_size, max_blocks;
  int kv_rows;                       // num_blocks * block_size: a box issued at this row lies past the cache (zeros)
};

SM90_DEVICE float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

SM90_DEVICE uint32_t pack2(float a, float b, bool bf16) {
  if (bf16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// accumulator registers 8 j .. 8 j + 7 (columns 16 j .. 16 j + 15) -> the A fragment of k-step j
template <int R> SM90_DEVICE void a_frag(const float (&v)[R], int j, bool bf16, uint32_t (&a)[4]) {
  a[0] = pack2(v[8 * j], v[8 * j + 1], bf16);
  a[1] = pack2(v[8 * j + 2], v[8 * j + 3], bf16);
  a[2] = pack2(v[8 * j + 4], v[8 * j + 5], bf16);
  a[3] = pack2(v[8 * j + 6], v[8 * j + 7], bf16);
}

// S (64 x 128, this warpgroup's query rows) = Q K^T, both K-major over D
template <int D>
SM90_DEVICE void mma_qk(float (&s)[64], uint32_t sq, uint32_t sk, bool bf16) {
  const uint64_t dq = make_smem_desc_sw128(sq, 16, 1024), dk = make_smem_desc_sw128(sk, 16, 1024);
#pragma unroll
  for (int k = 0; k < D / 16; ++k) {
    const uint32_t qo = (k >> 2) * (BLOCK_Q * 128) + (k & 3) * 32;
    const uint32_t ko = (k >> 2) * (BLOCK_KV * 128) + (k & 3) * 32;
    if (bf16) wgmma_ss_m64n128k16_bf16<0, 0>(s, advance_desc(dq, qo), advance_desc(dk, ko));
    else wgmma_ss_m64n128k16_f16<0, 0>(s, advance_desc(dq, qo), advance_desc(dk, ko));
  }
}

// O (64 x D) += P (registers, 64 x 128 keys) V (128 keys x D, MN-major: 64-column sub-tiles 16 KB apart)
template <int D>
SM90_DEVICE void mma_pv(float (&o)[D / 2], const float (&pr)[64], uint32_t sv, bool bf16) {
  const uint64_t dv = make_smem_desc_sw128(sv, BLOCK_KV * 128, 1024);
#pragma unroll
  for (int k = 0; k < BLOCK_KV / 16; ++k) {
    uint32_t a[4];
    a_frag(pr, k, bf16, a);
    const uint64_t b = advance_desc(dv, k * 2048);
    if constexpr (D == 128) {
      if (bf16) wgmma_rs_m64n128k16_bf16<1>(o, a, b);
      else wgmma_rs_m64n128k16_f16<1>(o, a, b);
    } else {
      if (bf16) wgmma_rs_m64n64k16_bf16<1>(o, a, b);
      else wgmma_rs_m64n64k16_f16<1>(o, a, b);
    }
  }
}

template <int D, bool EXTRA, bool BF16, bool PAGED>
__global__ void __launch_bounds__(NUM_THREADS, 1)
flash_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const FaParams p) {
  using C = FaCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem + C::Q_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_kv + KV_STAGES * C::KV_STAGE_BYTES);
  uint64_t* q_full = bars;                 // [1]
  uint64_t* kv_full = bars + 1;            // [2]
  uint64_t* kv_empty = bars + 3;           // [2]  one arrival per consumer warpgroup
  uint64_t* kv_land = bars + 5;            // [1]  the ragged last key tile, landed but not yet released

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int head = blockIdx.y;
  const int kv_head = head / (p.hq / p.hkv);
  int q_tile, seq_row0, len_q, len_k;
  int seq = 0;                                 // PAGED: the sequence of this CTA
  if (p.cu_seqlens != nullptr) {
    // packed batch: blockIdx.x enumerates (sequence, query tile) pairs in order; surplus CTAs (the grid is sized for
    // the worst case without knowing the lengths on the host) leave at once
    int t = (int)blockIdx.x, bsel = -1, start = 0, len = 0;
    for (int bb = 0; bb < p.batch; ++bb) {
      start = p.cu_seqlens[bb];
      len = p.cu_seqlens[bb + 1] - start;
      const int nt = (len + BLOCK_Q - 1) / BLOCK_Q;
      if (t < nt) { bsel = bb; break; }
      t -= nt;
    }
    if (bsel < 0) return;                      // uniform across the CTA: no barrier has been touched yet
    q_tile = t; seq_row0 = start; len_q = len; len_k = len;
    if constexpr (PAGED) { seq = bsel; len_k = p.seq_lens_k[bsel]; }
  } else {
    // heaviest (longest causal) query tiles first
    const int q_tiles = (p.seqlen_q + BLOCK_Q - 1) / BLOCK_Q;
    q_tile = p.causal ? (q_tiles - 1 - (int)blockIdx.x) : (int)blockIdx.x;
    seq_row0 = -1; len_q = p.seqlen_q; len_k = p.seqlen_k;
  }
  const int b = blockIdx.z;
  const int q_row0 = (seq_row0 >= 0 ? seq_row0 : b * p.seqlen_q) + q_tile * BLOCK_Q;   // row in the token-major Q / O
  const int kv_row0 = seq_row0 >= 0 ? seq_row0 : b * p.seqlen_k;
  const int kv_tiles_all = (len_k + BLOCK_KV - 1) / BLOCK_KV;
  // absolute position of the tile's first query row: PAGED rows follow the sequence's cached tokens (bottom-right
  // causal diagonal); otherwise queries and keys start together
  const int q_pos0 = (PAGED ? len_k - len_q : 0) + q_tile * BLOCK_Q;
  // causal: key tiles up to the one holding the tile's last row (q_tile when seqlen_q == seqlen_k); otherwise all
  const int kv_last = p.causal ? min(PAGED ? (q_pos0 + BLOCK_Q - 1) / BLOCK_KV + 1 : q_tile + 1, kv_tiles_all)
                               : kv_tiles_all;                                    // one past the last visible key tile
  // sliding window: the lowest key any row of this query tile can see is (q_pos0 - window + 1)
  const int kv_first = (EXTRA && p.window > 0) ? max(0, q_pos0 - p.window + 1) / BLOCK_KV : 0;
  const int kv_tiles = kv_last - kv_first;         // tiles walked; loop index j <-> key tile kv_first + j
  const bool resume = p.o_state != nullptr && p.has_prev != 0;   // block mode: continue from the stored state

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    mbar_init(kv_land, 1);
    fence_barrier_init();
  }
  if (warp == PRODUCER_WARP && lane == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_k);
    prefetch_tensormap(&tmap_v);
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // ================================================================ TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, C::Q_BYTES);
#pragma unroll
      for (int h = 0; h < D / 64; ++h)                     // boxes [128 rows, 64 d] -> K-major swizzled sub-tiles
        tma_load_2d(&tmap_q, q_full, smem_q + h * (BLOCK_Q * 128), head * D + h * 64, q_row0);
    }
    const bool ragged = (len_k % BLOCK_KV) != 0 && kv_last == kv_tiles_all;   // the walk ends on a partial key tile
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < kv_tiles; ++j) {
      mbar_wait(&kv_empty[stage], phase ^ 1);
      uint8_t* sk = smem_kv + stage * C::KV_STAGE_BYTES;
      uint8_t* sv = sk + C::K_BYTES;
      // The rows of a ragged last key tile past the sequence's keys hold another sequence's rows (the tensor maps span
      // the whole packed / batched tensor) or a paged block's unwritten tail slots.  Their P is 0, but 0 * NaN or Inf
      // in the P V MMA is NaN.  So that tile lands on kv_land instead: this warp zeroes those V rows (128-byte rows of
      // each 64-column sub-tile, whatever the swizzle) and only then releases the stage to the consumers.
      const bool clean = ragged && j == kv_tiles - 1;
      uint64_t* full = clean ? kv_land : &kv_full[stage];
      if constexpr (PAGED) {
        // the 128-key tile is assembled from 128 / block_size boxes of block_size rows, one per lane; every box is a
        // whole number of 1024-byte swizzle atoms, so the stage has the layout one 128-row box gives.  Boxes of blocks
        // past the sequence's last one are issued past the end of the cache: TMA fills them with zeros (same byte
        // count), and their table entries are never read.
        if (lane == 0) mbar_arrive_expect_tx(full, C::KV_STAGE_BYTES);
        __syncwarp();
        const int bs = p.block_size;
        if (lane < BLOCK_KV / bs) {
          const int key = (kv_first + j) * BLOCK_KV + lane * bs;
          const int kb = key / bs;
          int row = p.kv_rows;
          if (key < len_k && kb < p.max_blocks) {
            const int blk = p.block_tables[(size_t)seq * p.max_blocks + kb];
            if (blk >= 0) row = blk * bs;
          }
#pragma unroll
          for (int h = 0; h < D / 64; ++h) {
            tma_load_2d(&tmap_k, full, sk + h * (BLOCK_KV * 128) + lane * bs * 128, kv_head * D + h * 64, row);
            tma_load_2d(&tmap_v, full, sv + h * (BLOCK_KV * 128) + lane * bs * 128, kv_head * D + h * 64, row);
          }
        }
      } else if (lane == 0) {
        mbar_arrive_expect_tx(full, C::KV_STAGE_BYTES);
        const int row = kv_row0 + (kv_first + j) * BLOCK_KV;
#pragma unroll
        for (int h = 0; h < D / 64; ++h) {
          tma_load_2d(&tmap_k, full, sk + h * (BLOCK_KV * 128), kv_head * D + h * 64, row);
          tma_load_2d(&tmap_v, full, sv + h * (BLOCK_KV * 128), kv_head * D + h * 64, row);
        }
      }
      __syncwarp();
      if (clean) {
        mbar_wait(kv_land, 0);
        const int r0 = len_k - (kv_tiles_all - 1) * BLOCK_KV;
        const int per_sub = (BLOCK_KV - r0) * 8;                       // 16-byte chunks past row r0 in one sub-tile
#pragma unroll 1
        for (int i = lane; i < per_sub * (D / 64); i += 32) {
          const int h = i / per_sub;
          *reinterpret_cast<uint4*>(sv + r0 * 128 + h * (BLOCK_KV * 128) + (i - h * per_sub) * 16) =
              make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async();                                           // generic writes -> the wgmma (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&kv_full[stage]);
      }
      if (++stage == KV_STAGES) { stage = 0; phase ^= 1; }
    }
    return;
  }

  // ================================================================ consumers: thread owns 2 query rows
  constexpr bool bf16 = BF16;
  const int wg = threadIdx.x >> 7;
  const int wrow = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // row inside the tile for h = 0 (h = 1: + 8)
  const int cq = 2 * (lane & 3);                                  // column offset inside every 8-column group
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};                        // running max, exp2 domain
  float l_run[2] = {0.f, 0.f};
  if (resume) {
    // resume from the merged result of the key blocks processed by earlier launches (normalised output + LSE)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = wrow + 8 * h;
      const size_t row_ = (size_t)q_row0 + r;
      float lse_prev = -INFINITY;
      if (q_tile * BLOCK_Q + r < len_q) lse_prev = p.lse[row_ * p.hq + head];
      if (lse_prev > -INFINITY) {
        m_run[h] = lse_prev * LOG2E;
        l_run[h] = (lane & 3) == 0 ? 1.f : 0.f;   // the 4 lanes of a row hold partial sums, added at the end
        const float* src = p.o_state + row_ * ((size_t)p.hq * D) + (size_t)head * D;
#pragma unroll
        for (int c = 0; c < D / 8; ++c) {
          const float2 t2 = *reinterpret_cast<const float2*>(src + 8 * c + cq);
          o[4 * c + 2 * h] = t2.x;
          o[4 * c + 2 * h + 1] = t2.y;
        }
      }
    }
  }
  const float slope2 = (EXTRA && p.alibi != nullptr) ? p.alibi[head] * LOG2E : 0.f;
  const uint32_t sq = smem_u32(smem_q) + wg * 64 * 128;
  mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < kv_tiles; ++j) {
    mbar_wait(&kv_full[stage], phase);
    const uint32_t sk = smem_u32(smem_kv + stage * C::KV_STAGE_BYTES);
    float s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
    wgmma_fence();
    mma_qk<D>(s, sq, sk, bf16);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    const int kt = kv_first + j;
    const int k_base = kt * BLOCK_KV;
    // PAGED (always causal): a tile is masked when its last key lies after the tile's first query row.  Every query
    // row sits before the end of its sequence's keys, so that also covers a ragged last tile, and k_lim = q_pos.
    const bool masked = PAGED ? (k_base + BLOCK_KV - 1 > q_pos0) || (EXTRA && p.window > 0)
                              : (p.causal && kt == q_tile) || (kt == kv_tiles_all - 1 && (len_k % BLOCK_KV) != 0) ||
                                    (EXTRA && p.window > 0);
    float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int h = (i >> 1) & 1;
      const int q_pos = q_pos0 + wrow + 8 * h;
      const int key = k_base + 8 * (i >> 2) + cq + (i & 1);
      float x = s[i] * p.scale_log2;
      if (EXTRA) x = fmaf(slope2, (float)(key - q_pos), x);
      if (masked) {
        const int k_lim = PAGED ? q_pos : (p.causal && kt == q_tile) ? min(q_pos, len_k - 1) : len_k - 1;
        if (key > k_lim || (EXTRA && p.window > 0 && key < q_pos - p.window + 1)) x = -INFINITY;
      }
      s[i] = x;
      mt[h] = fmaxf(mt[h], x);
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 1));
      mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 2));
      const float m_new = fmaxf(m_run[h], mt[h]);
      alpha[h] = m_new == -INFINITY ? 1.f : fast_exp2(m_run[h] - m_new);
      m_use[h] = m_new == -INFINITY ? 0.f : m_new;
      m_run[h] = m_new;
      l_run[h] *= alpha[h];
    }
    float lt[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int h = (i >> 1) & 1;
      const float e = fast_exp2(s[i] - m_use[h]);
      s[i] = e;
      lt[h] += e;
    }
    l_run[0] += lt[0];
    l_run[1] += lt[1];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    wgmma_fence();
    mma_pv<D>(o, s, sk + C::K_BYTES, bf16);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[stage]);   // K_j / V_j consumed
    if (++stage == KV_STAGES) { stage = 0; phase ^= 1; }
  }
  // ---- epilogue: full row sums (4 lanes share a row), normalise and store this thread's two rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wrow + 8 * h;
    if (q_tile * BLOCK_Q + r >= len_q) continue;          // rows past the end of a (packed) sequence are never stored
    const size_t row = (size_t)q_row0 + r;
    const float inv_l = l_run[h] > 0.f ? 1.f / l_run[h] : 0.f;
    if (p.o_state != nullptr) {
      float* dst = p.o_state + row * ((size_t)p.hq * D) + (size_t)head * D;
#pragma unroll
      for (int c = 0; c < D / 8; ++c)
        *reinterpret_cast<float2*>(dst + 8 * c + cq) = make_float2(o[4 * c + 2 * h] * inv_l, o[4 * c + 2 * h + 1] * inv_l);
    } else {
      uint8_t* dst = reinterpret_cast<uint8_t*>(p.out) + (row * ((size_t)p.hq * D) + (size_t)head * D) * 2;
#pragma unroll
      for (int c = 0; c < D / 8; ++c)
        *reinterpret_cast<uint32_t*>(dst + (8 * c + cq) * 2) = pack2(o[4 * c + 2 * h] * inv_l, o[4 * c + 2 * h + 1] * inv_l, bf16);
    }
    if (p.lse && (lane & 3) == 0)
      p.lse[row * p.hq + head] = l_run[h] > 0.f ? (m_run[h] + log2f(l_run[h])) * 0.6931471805599453f : -INFINITY;
  }
}

template <int D>
int launch_flash_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int batch, int seqlen_q,
                     int seqlen_k, int hq, int hkv, int causal, float scale, int dtype, cudaStream_t stream,
                     const int* cu_seqlens, long long total_tokens, float* o_state, int has_prev, int window,
                     const float* alibi, const int* block_tables, const int* seq_lens_k, int block_size,
                     int max_blocks, int num_blocks) {
  using C = FaCfg<D>;
  const bool bf16 = dtype == CB_BF16;
  const bool paged = block_tables != nullptr;
  CUtensorMap tq, tk, tv;
  const uint64_t rows_q = cu_seqlens ? (uint64_t)total_tokens : (uint64_t)batch * seqlen_q;
  const uint64_t rows_k = paged ? (uint64_t)num_blocks * block_size
                                : cu_seqlens ? (uint64_t)total_tokens : (uint64_t)batch * seqlen_k;
  const uint32_t box_k = paged ? (uint32_t)block_size : BLOCK_KV;
  int r = make_tmap_2d_16b(&tq, q, rows_q, (uint64_t)hq * D, (uint64_t)hq * D, BLOCK_Q, 64, bf16);
  if (r) return 1000 + r;
  r = make_tmap_2d_16b(&tk, k, rows_k, (uint64_t)hkv * D, (uint64_t)hkv * D, box_k, 64, bf16);
  if (r) return 2000 + r;
  r = make_tmap_2d_16b(&tv, v, rows_k, (uint64_t)hkv * D, (uint64_t)hkv * D, box_k, 64, bf16);
  if (r) return 3000 + r;
  FaParams p;
  p.cu_seqlens = cu_seqlens;
  p.o_state = o_state; p.has_prev = has_prev;
  p.batch = batch; p.seqlen_q = seqlen_q; p.seqlen_k = seqlen_k; p.hq = hq; p.hkv = hkv; p.causal = causal;
  p.scale_log2 = scale * LOG2E;
  p.out = out; p.lse = lse; p.out_dtype = dtype;
  p.window = window; p.alibi = alibi;
  p.block_tables = block_tables; p.seq_lens_k = seq_lens_k; p.block_size = block_size; p.max_blocks = max_blocks;
  p.kv_rows = paged ? num_blocks * block_size : 0;
  static bool attr_set = false;
  if (!attr_set) {
    const void* fns[8] = {
        (const void*)flash_fwd_kernel<D, false, true, false>, (const void*)flash_fwd_kernel<D, true, true, false>,
        (const void*)flash_fwd_kernel<D, false, false, false>, (const void*)flash_fwd_kernel<D, true, false, false>,
        (const void*)flash_fwd_kernel<D, false, true, true>, (const void*)flash_fwd_kernel<D, true, true, true>,
        (const void*)flash_fwd_kernel<D, false, false, true>, (const void*)flash_fwd_kernel<D, true, false, true>};
    for (const void* f : fns) {
      cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
      if (e != cudaSuccess) return (int)e;
    }
    attr_set = true;
  }
  // packed: at most total/128 + batch query tiles exist; uniform: ceil(seqlen / 128) per sequence
  dim3 grid(cu_seqlens ? (unsigned)(total_tokens / BLOCK_Q + batch) : (unsigned)((seqlen_q + BLOCK_Q - 1) / BLOCK_Q), hq,
            cu_seqlens ? 1 : batch);
  const bool extra = window > 0 || alibi != nullptr;
  decltype(&flash_fwd_kernel<D, false, false, false>) kern;
  if (paged) {
    kern = extra ? (bf16 ? flash_fwd_kernel<D, true, true, true> : flash_fwd_kernel<D, true, false, true>)
                 : (bf16 ? flash_fwd_kernel<D, false, true, true> : flash_fwd_kernel<D, false, false, true>);
  } else {
    kern = extra ? (bf16 ? flash_fwd_kernel<D, true, true, false> : flash_fwd_kernel<D, true, false, false>)
                 : (bf16 ? flash_fwd_kernel<D, false, true, false> : flash_fwd_kernel<D, false, false, false>);
  }
  kern<<<grid, NUM_THREADS, C::SMEM_BYTES, stream>>>(tq, tk, tv, p);
  return (int)cudaGetLastError();
}


// =====================================================================================================================
// Flash attention BACKWARD on wgmma.
//
//   P = exp(scale * Q K^T - LSE),  dP = dO V^T,  dS = P o (dP - delta),  delta = rowsum(dO o O)
//   dV = P^T dO,   dK = scale * dS^T Q,   dQ = scale * dS K
//
// One CTA owns ONE key tile (128 keys) of ONE kv head and walks over every query tile (64 rows) of every query head of
// its GQA group that can see it.  dK / dV therefore accumulate in registers across the whole walk - over the query
// tiles AND over the query heads of the group - and are written exactly once (no atomics, no KV expansion); dQ leaves
// the CTA as fp32 reductions into an accumulator that a cast kernel turns into bf16/fp16 afterwards.
//
// Each consumer warpgroup owns 64 of the keys and computes everything TRANSPOSED so that its rows are keys:
//   S^T = K Q^T and dP^T = V dO^T   [64 keys x 64 q]   (shared-memory operands, K-major over D)
//   dV += P^T dO,  dK += dS^T Q    (P^T / dS^T straight from registers as the A operand, dO / Q MN-major)
//   dQ  = dS K                      (dS^T of both warpgroups written to shared memory and read MN-major as A; each
//                                    warpgroup computes 64 of the 128 head-dim columns, K read MN-major as B)
// Warp 8 is the TMA producer (K, V once; Q_i / dO_i through a 2-stage ring).
// Shared memory: K 32 KB + V 32 KB + 2 x (Q 16 KB + dO 16 KB) + dS^T 16 KB = 144 KB (D = 128).
constexpr int BWD_BLOCK_KV = 128;
constexpr int BWD_BLOCK_Q = 64;
constexpr int BWD_QSTAGES = 2;

template <int D> struct FaBwdCfg {
  static constexpr int K_BYTES = BWD_BLOCK_KV * D * 2;
  static constexpr int V_BYTES = BWD_BLOCK_KV * D * 2;
  static constexpr int Q_BYTES = BWD_BLOCK_Q * D * 2;
  static constexpr int DO_BYTES = BWD_BLOCK_Q * D * 2;
  static constexpr int QDO_STAGE_BYTES = Q_BYTES + DO_BYTES;
  static constexpr int DS_BYTES = BWD_BLOCK_KV * BWD_BLOCK_Q * 2;
  static constexpr int SMEM_BYTES = K_BYTES + V_BYTES + BWD_QSTAGES * QDO_STAGE_BYTES + DS_BYTES + 1024 /*align*/ +
                                    256 /*barriers*/;
};

struct FaBwdParams {
  const int* cu_seqlens;             // packed batch boundaries (see FaParams) or null
  int batch, seqlen;                 // equal-length sequences, seqlen_q == seqlen_k (self attention)
  int hq, hkv;
  int causal;
  float scale, scale_log2;
  const float* lse;                  // [batch * seqlen, hq] natural log
  const float* delta;                // [batch * seqlen, hq] rowsum(dO o O)
  float* dq_acc;                     // [batch * seqlen, hq * D] fp32, zero-initialised
  void* dk;                          // [batch * seqlen, hkv * D]
  void* dv;
  // ring attention: dK / dV of this key block are ADDED (fp32 reductions) into accumulators that may live in the block
  // owner's memory (peer-mapped symmetric buffer: the reduction crosses NVLink) instead of being stored
  float* dk_acc;                     // [rows, hkv * D] fp32 or null
  float* dv_acc;
  int out_dtype;
};

SM90_DEVICE void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// [64 keys x 64 q] = X (this warpgroup's 64 key rows, K-major over D) x Y^T (64 q rows, K-major over D)
template <int D>
SM90_DEVICE void mma_kq(float (&s)[32], uint32_t sx, uint32_t sy, bool bf16) {
  const uint64_t dx = make_smem_desc_sw128(sx, 16, 1024), dy = make_smem_desc_sw128(sy, 16, 1024);
#pragma unroll
  for (int k = 0; k < D / 16; ++k) {
    const uint32_t xo = (k >> 2) * (BWD_BLOCK_KV * 128) + (k & 3) * 32;
    const uint32_t yo = (k >> 2) * (BWD_BLOCK_Q * 128) + (k & 3) * 32;
    if (bf16) wgmma_ss_m64n64k16_bf16<0, 0>(s, advance_desc(dx, xo), advance_desc(dy, yo));
    else wgmma_ss_m64n64k16_f16<0, 0>(s, advance_desc(dx, xo), advance_desc(dy, yo));
  }
}

// [64 keys x D] += A (registers: [64 keys x 64 q]) x Y (64 q rows x D, MN-major: 64-column sub-tiles 8 KB apart)
template <int D>
SM90_DEVICE void mma_acc(float (&acc)[D / 2], const float (&a_regs)[32], uint32_t sy, bool bf16) {
  static_assert(D == 128, "head_dim 128");
  const uint64_t dy = make_smem_desc_sw128(sy, BWD_BLOCK_Q * 128, 1024);
#pragma unroll
  for (int k = 0; k < BWD_BLOCK_Q / 16; ++k) {
    uint32_t a[4];
    a_frag(a_regs, k, bf16, a);
    if (bf16) wgmma_rs_m64n128k16_bf16<1>(acc, a, advance_desc(dy, k * 2048));
    else wgmma_rs_m64n128k16_f16<1>(acc, a, advance_desc(dy, k * 2048));
  }
}

template <int D, bool BF16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
flash_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                 const FaBwdParams p) {
  using C = FaBwdCfg<D>;
  static_assert(D == 128, "head_dim 128");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_k = smem;
  uint8_t* smem_v = smem_k + C::K_BYTES;
  uint8_t* smem_qdo = smem_v + C::V_BYTES;
  uint8_t* smem_ds = smem_qdo + BWD_QSTAGES * C::QDO_STAGE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_ds + C::DS_BYTES);
  uint64_t* kv_full = bars;                // [1]
  uint64_t* qdo_full = bars + 1;           // [2]
  uint64_t* qdo_empty = bars + 3;          // [2]  one arrival per consumer warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int kv_head = blockIdx.y;
  const int group = p.hq / p.hkv;
  int kv_tile, seq_row0, len;
  if (p.cu_seqlens != nullptr) {
    int t = (int)blockIdx.x, bsel = -1, start = 0;
    len = 0;
    for (int bb = 0; bb < p.batch; ++bb) {
      start = p.cu_seqlens[bb];
      len = p.cu_seqlens[bb + 1] - start;
      const int nt = (len + BWD_BLOCK_KV - 1) / BWD_BLOCK_KV;
      if (t < nt) { bsel = bb; break; }
      t -= nt;
    }
    if (bsel < 0) return;
    kv_tile = t; seq_row0 = start;
  } else {
    kv_tile = blockIdx.x; seq_row0 = (int)blockIdx.z * p.seqlen; len = p.seqlen;
  }
  const int q_tiles = (len + BWD_BLOCK_Q - 1) / BWD_BLOCK_Q;
  // causal: query tile i (rows 64 i ..) sees key tile j (keys 128 j ..) iff 64 i + 63 >= 128 j  <=>  i >= 2 j
  const int i_start = p.causal ? 2 * kv_tile : 0;
  const int n_i = max(q_tiles - i_start, 0);
  const int n_iter = n_i * group;                                  // (query head of the group, query tile) pairs
  const int kv_row0 = seq_row0 + kv_tile * BWD_BLOCK_KV;
  const bool ragged = (len % BWD_BLOCK_KV) != 0;                    // partial last key tile and / or query tile

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int i = 0; i < BWD_QSTAGES; ++i) {
      mbar_init(&qdo_full[i], 1);
      mbar_init(&qdo_empty[i], 2);
    }
    fence_barrier_init();
  }
  if (warp == PRODUCER_WARP && lane == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_k);
    prefetch_tensormap(&tmap_v);
    prefetch_tensormap(&tmap_do);
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // ================================================================ TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(kv_full, C::K_BYTES + C::V_BYTES);
#pragma unroll
      for (int h = 0; h < D / 64; ++h) {
        tma_load_2d(&tmap_k, kv_full, smem_k + h * (BWD_BLOCK_KV * 128), kv_head * D + h * 64, kv_row0);
        tma_load_2d(&tmap_v, kv_full, smem_v + h * (BWD_BLOCK_KV * 128), kv_head * D + h * 64, kv_row0);
      }
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < n_iter; ++it) {
      mbar_wait(&qdo_empty[stage], phase ^ 1);
      if (lane == 0) {
        const int hq = kv_head * group + it / n_i;
        const int q_row0 = seq_row0 + (i_start + it % n_i) * BWD_BLOCK_Q;
        uint8_t* sq = smem_qdo + stage * C::QDO_STAGE_BYTES;
        uint8_t* sdo = sq + C::Q_BYTES;
        mbar_arrive_expect_tx(&qdo_full[stage], C::QDO_STAGE_BYTES);
#pragma unroll
        for (int h = 0; h < D / 64; ++h) {
          tma_load_2d(&tmap_q, &qdo_full[stage], sq + h * (BWD_BLOCK_Q * 128), hq * D + h * 64, q_row0);
          tma_load_2d(&tmap_do, &qdo_full[stage], sdo + h * (BWD_BLOCK_Q * 128), hq * D + h * 64, q_row0);
        }
      }
      __syncwarp();
      if (++stage == BWD_QSTAGES) { stage = 0; phase ^= 1; }
    }
    return;
  }

  // ================================================================ consumers: thread owns 2 key rows
  constexpr bool bf16 = BF16;
  const int wg = threadIdx.x >> 7;
  const int krow = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // key row inside the tile for h = 0 (h = 1: + 8)
  const int cq = 2 * (lane & 3);
  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  const uint32_t sk = smem_u32(smem_k), sv = smem_u32(smem_v), sds = smem_u32(smem_ds);
  if (n_iter > 0) mbar_wait(kv_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < n_iter; ++it) {
    const int hq = kv_head * group + it / n_i;
    const int q_tile = i_start + it % n_i;
    const int q_row0 = seq_row0 + q_tile * BWD_BLOCK_Q;
    const int q_base = q_tile * BWD_BLOCK_Q;
    // per-query statistics of this thread's 16 columns (rows past the end of the sequence read as 0; their P / dS
    // are forced to 0 below)
    float lse2[16], dlt[16];
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * c + cq + e;
        const bool live = q_base + col < len;
        const size_t idx = (size_t)(q_row0 + col) * p.hq + hq;
        lse2[2 * c + e] = live ? __ldg(p.lse + idx) * LOG2E : 0.f;
        dlt[2 * c + e] = live ? __ldg(p.delta + idx) : 0.f;
      }
    mbar_wait(&qdo_full[stage], phase);
    const uint32_t sq = smem_u32(smem_qdo + stage * C::QDO_STAGE_BYTES);
    const uint32_t sdo = sq + C::Q_BYTES;
    float st[32], dpt[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { st[i] = 0.f; dpt[i] = 0.f; }
    wgmma_fence();
    mma_kq<D>(st, sk + wg * 64 * 128, sq, bf16);
    mma_kq<D>(dpt, sv + wg * 64 * 128, sdo, bf16);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(st);
    reg_fence(dpt);
    const bool diag = (p.causal && (q_tile <= 2 * kv_tile + 1)) ||
                      (ragged && (kv_tile == (len - 1) / BWD_BLOCK_KV || q_tile == q_tiles - 1));
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int h = (i >> 1) & 1;
      const int key_pos = kv_tile * BWD_BLOCK_KV + krow + 8 * h;
      const int ci = 2 * (i >> 2) + (i & 1);                 // index into lse2 / dlt
      const int qp = q_base + 8 * (i >> 2) + cq + (i & 1);
      float pe = fast_exp2(st[i] * p.scale_log2 - lse2[ci]);
      float de = pe * (dpt[i] - dlt[ci]);
      if (diag && !(key_pos < len && qp >= (p.causal ? key_pos : 0) && qp < len)) { pe = 0.f; de = 0.f; }
      st[i] = pe;
      dpt[i] = de;
    }
    // dS^T of both warpgroups -> shared memory ([128 keys x 64 q], 128-byte rows, SWIZZLE_128B); the previous
    // iteration's dQ MMAs of BOTH warpgroups have retired (each waited for its own before its dQ reductions)
    named_sync(1, 256);
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const int r = krow + 8 * h;
      const int col = 8 * (i >> 2) + cq;
      *reinterpret_cast<uint32_t*>(smem_ds + r * 128 + (((col >> 3) ^ (r & 7)) << 4) + (col & 7) * 2) =
          pack2(dpt[i], dpt[i + 1], bf16);
    }
    fence_proxy_async();
    named_sync(1, 256);
    float dq[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] = 0.f;
    wgmma_fence();
    mma_acc<D>(dv, st, sdo, bf16);
    mma_acc<D>(dk, dpt, sq, bf16);
    {
      // dQ [64 q x 64 d (columns 64 wg ..)] = dS (MN-major view of dS^T) x K (MN-major: sub-tile wg of the K tile)
      const uint64_t da = make_smem_desc_sw128(sds, 8192, 1024);
      const uint64_t db = make_smem_desc_sw128(sk + wg * (BWD_BLOCK_KV * 128), 8192, 1024);
#pragma unroll
      for (int k = 0; k < BWD_BLOCK_KV / 16; ++k) {
        if (bf16) wgmma_ss_m64n64k16_bf16<1, 1>(dq, advance_desc(da, k * 2048), advance_desc(db, k * 2048));
        else wgmma_ss_m64n64k16_f16<1, 1>(dq, advance_desc(da, k * 2048), advance_desc(db, k * 2048));
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dv);
    reg_fence(dk);
    reg_fence(dq);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&qdo_empty[stage]);     // Q_i / dO_i consumed
    if (++stage == BWD_QSTAGES) { stage = 0; phase ^= 1; }
    // dQ rows: query q_base + 16 w' + l / 4 (+ 8), columns 64 wg + 8 c + cq (+ 1)
    const size_t row_stride = (size_t)p.hq * D;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int qr = (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (q_base + qr >= len) continue;
      float* dst = p.dq_acc + (size_t)(q_row0 + qr) * row_stride + (size_t)hq * D + wg * 64 + cq;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        atomicAdd(dst + 8 * c, dq[4 * c + 2 * h] * p.scale);
        atomicAdd(dst + 8 * c + 1, dq[4 * c + 2 * h + 1] * p.scale);
      }
    }
  }
  // ---- epilogue: dV and scale * dK rows of this thread's keys
  const size_t ld = (size_t)p.hkv * D;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = krow + 8 * h;
    if (kv_tile * BWD_BLOCK_KV + r >= len) continue;       // a ragged last tile leaves some rows without a key
    const size_t off = ((size_t)kv_row0 + r) * ld + (size_t)kv_head * D + cq;
#pragma unroll
    for (int c = 0; c < D / 8; ++c) {
      const float v0 = dv[4 * c + 2 * h], v1 = dv[4 * c + 2 * h + 1];
      const float k0 = dk[4 * c + 2 * h] * p.scale, k1 = dk[4 * c + 2 * h + 1] * p.scale;
      if (p.dk_acc != nullptr) {
        if (n_iter > 0) {
          atomicAdd(p.dv_acc + off + 8 * c, v0);
          atomicAdd(p.dv_acc + off + 8 * c + 1, v1);
          atomicAdd(p.dk_acc + off + 8 * c, k0);
          atomicAdd(p.dk_acc + off + 8 * c + 1, k1);
        }
      } else {
        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.dv) + (off + 8 * c) * 2) = pack2(v0, v1, bf16);
        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.dk) + (off + 8 * c) * 2) = pack2(k0, k1, bf16);
      }
    }
  }
}

// delta[t, h] = sum_d dO[t, h, d] * O[t, h, d]   (one warp per (token, head) row)
template <typename T>
__global__ void flash_bwd_delta_kernel(const T* __restrict__ out, const T* __restrict__ dout, float* __restrict__ delta,
                                       long long rows, int D) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const T* o = out + row * D;
  const T* g = dout + row * D;
  float acc = 0.f;
  for (int i = lane * 8; i < D; i += 32 * 8) {
    Vec16<T> a, b2;
    a.load(o + i);
    b2.load(g + i);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc += a.get(e) * b2.get(e);
  }
  acc = warp_sum(acc);
  if (lane == 0) delta[row] = acc;
}

template <typename T>
__global__ void flash_bwd_cast_dq_kernel(const float* __restrict__ acc, T* __restrict__ dq, long long n) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= n) return;
  const float4 a = *reinterpret_cast<const float4*>(acc + i);
  const float4 b2 = *reinterpret_cast<const float4*>(acc + i + 4);
  Vec16<T> o;
  o.set(0, a.x); o.set(1, a.y); o.set(2, a.z); o.set(3, a.w);
  o.set(4, b2.x); o.set(5, b2.y); o.set(6, b2.z); o.set(7, b2.w);
  o.store(dq + i);
}

template <int D>
int launch_flash_bwd(const void* q, const void* k, const void* v, const void* dout, const float* lse, const float* delta,
                     float* dq_acc, void* dk, void* dv, int batch, int seqlen, int hq, int hkv, int causal, float scale,
                     int dtype, cudaStream_t stream, const int* cu_seqlens = nullptr, long long total_tokens = 0,
                     float* dk_acc = nullptr, float* dv_acc = nullptr) {
  using C = FaBwdCfg<D>;
  const bool bf16 = dtype == CB_BF16;
  CUtensorMap tq, tk, tv, tdo;
  const uint64_t T = cu_seqlens ? (uint64_t)total_tokens : (uint64_t)batch * seqlen;
  int r = make_tmap_2d_16b(&tq, q, T, (uint64_t)hq * D, (uint64_t)hq * D, BWD_BLOCK_Q, 64, bf16);
  if (r) return 1000 + r;
  r = make_tmap_2d_16b(&tdo, dout, T, (uint64_t)hq * D, (uint64_t)hq * D, BWD_BLOCK_Q, 64, bf16);
  if (r) return 4000 + r;
  r = make_tmap_2d_16b(&tk, k, T, (uint64_t)hkv * D, (uint64_t)hkv * D, BWD_BLOCK_KV, 64, bf16);
  if (r) return 2000 + r;
  r = make_tmap_2d_16b(&tv, v, T, (uint64_t)hkv * D, (uint64_t)hkv * D, BWD_BLOCK_KV, 64, bf16);
  if (r) return 3000 + r;
  FaBwdParams p;
  p.cu_seqlens = cu_seqlens;
  p.batch = batch; p.seqlen = seqlen; p.hq = hq; p.hkv = hkv; p.causal = causal;
  p.scale = scale; p.scale_log2 = scale * LOG2E;
  p.lse = lse; p.delta = delta; p.dq_acc = dq_acc; p.dk = dk; p.dv = dv; p.out_dtype = dtype;
  p.dk_acc = dk_acc; p.dv_acc = dv_acc;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(flash_bwd_kernel<D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(flash_bwd_kernel<D, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  dim3 grid(cu_seqlens ? (unsigned)(total_tokens / BWD_BLOCK_KV + batch) : (unsigned)((seqlen + BWD_BLOCK_KV - 1) / BWD_BLOCK_KV),
            hkv, cu_seqlens ? 1 : batch);
  if (bf16) flash_bwd_kernel<D, true><<<grid, NUM_THREADS, C::SMEM_BYTES, stream>>>(tq, tk, tv, tdo, p);
  else flash_bwd_kernel<D, false><<<grid, NUM_THREADS, C::SMEM_BYTES, stream>>>(tq, tk, tv, tdo, p);
  return (int)cudaGetLastError();
}

// dtype validated by the caller (bf16 or fp16)
int launch_flash_delta(const void* out, const void* dout, float* delta, long long rows, int head_dim, int dtype,
                       cudaStream_t stream) {
  const int wpb = 8;
  const unsigned blocks = (unsigned)((rows + wpb - 1) / wpb);
  if (dtype == CB_BF16)
    flash_bwd_delta_kernel<__nv_bfloat16><<<blocks, wpb * 32, 0, stream>>>(
        (const __nv_bfloat16*)out, (const __nv_bfloat16*)dout, delta, rows, head_dim);
  else
    flash_bwd_delta_kernel<__half><<<blocks, wpb * 32, 0, stream>>>((const __half*)out, (const __half*)dout, delta,
                                                                    rows, head_dim);
  return (int)cudaGetLastError();
}

// the envelope of the wgmma backward kernel, shared by both backward entry points
bool bwd_args_ok(int hq, int hkv, int head_dim, int dtype) {
  return hkv > 0 && hq % hkv == 0 && head_dim == 128 && (dtype == CB_BF16 || dtype == CB_F16);
}

}  // namespace

extern "C" {

// The one forward entry point.  q [rows_q, hq, D], k / v [rows_k, hkv, D] contiguous token-major, 16-byte aligned
// bases; out like q; lse [rows_q, hq] fp32 natural log (may be null except in block mode).  Sequence lengths need not
// be multiples of the tile: partial tiles are masked (keys) / not stored (queries).  The arguments select the mode:
//   uniform : cu_seqlens null, `batch` sequences of seqlen_q queries / seqlen_k keys (causal => seqlen_q == seqlen_k);
//   packed  : cu_seqlens int32[batch + 1] ON THE DEVICE, self attention over `total_tokens` rows (seqlen_q / seqlen_k
//             ignored).  The host never reads the boundaries: the grid is sized for the worst case and surplus CTAs
//             exit.  Reference counterpart: `flash_attn_varlen_kvpacked_func` behind
//             `extensions/pybind/flash_attention/flash_attention_dao_cuda.py:37-96`;
//   prefill : packed and causal with a sliding window (`window` > 0: query q sees keys (q - window, q]; Mistral) and /
//             or ALiBi slopes (`alibi` [hq] fp32: score += slope * (key - query); BLOOM, Baichuan-13B);
//   block   : o_state non-null, uniform only (ring attention, see below): the fp32 online-softmax state (o_state
//             [rows_q, hq, D], lse) is written instead of `out`, and read first when `has_prev`;
//   paged   : block_tables non-null, packed and causal, no o_state (prefill after a prefix-cache hit, and the building
//             block of chunked prefill): k / v are the paged caches [num_blocks, block_size, hkv, D] (block_size 8, 16,
//             32, 64 or 128).  Sequence b's new query rows sit at the absolute positions seq_lens_k[b] - n_b ..
//             seq_lens_k[b] - 1 (n_b from cu_seqlens) and see the keys 0 .. seq_lens_k[b] - 1 through
//             block_tables[b] (int32 [batch, max_blocks]); window / alibi apply on absolute positions.  seq_lens_k and
//             block_tables live ON THE DEVICE and are never read by the host; entries past a sequence's last block
//             are never read (they may be -1 or stale).  lse may be null.
// Anything outside that envelope returns cudaErrorInvalidValue and launches nothing.
// Sequences do not see each other: the out / lse rows of a sequence (a packed sequence, a batch entry of a uniform
// call, a paged sequence) depend only on that sequence's q / k / v rows, even where other rows hold NaN or Inf: a
// ragged last key tile zeroes its V rows past the sequence's keys, and a paged sequence's unwritten tail slots need
// not be finite.  As in flash-attn 2, keys a causal row must not see INSIDE its own sequence's diagonal tile are masked
// to p = 0 but still enter the P V MMA, so a NaN / Inf value in a future key of the same sequence reaches earlier rows.
int cb_flash_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, float* o_state, int has_prev,
                      const int* cu_seqlens, long long total_tokens, int batch, int seqlen_q, int seqlen_k, int hq,
                      int hkv, int head_dim, int causal, float scale, int window, const float* alibi,
                      const int* block_tables, const int* seq_lens_k, int block_size, int max_blocks, int num_blocks,
                      int dtype, cudaStream_t stream) {
  const bool packed = cu_seqlens != nullptr;
  const bool paged = block_tables != nullptr;
  const bool block_size_ok = block_size == 8 || block_size == 16 || block_size == 32 || block_size == 64 ||
                             block_size == 128;
  if ((dtype != CB_BF16 && dtype != CB_F16) || hkv <= 0 || hq % hkv || (head_dim != 64 && head_dim != 128) ||
      (!packed && causal && seqlen_q != seqlen_k) || window < 0 || ((window > 0 || alibi) && !(packed && causal)) ||
      (o_state ? (packed || lse == nullptr) : has_prev != 0) ||
      (paged ? !(packed && causal && o_state == nullptr && seq_lens_k != nullptr && block_size_ok && max_blocks > 0 &&
                 num_blocks > 0 && (long long)num_blocks * block_size <= 0x7fffffffLL)
             : seq_lens_k != nullptr))
    return (int)cudaErrorInvalidValue;
  if (batch <= 0 || (packed ? total_tokens <= 0 : seqlen_q <= 0)) return 0;
  return (head_dim == 128 ? launch_flash_fwd<128> : launch_flash_fwd<64>)(
      q, k, v, out, lse, batch, seqlen_q, seqlen_k, hq, hkv, causal, scale, dtype, stream, cu_seqlens, total_tokens,
      o_state, has_prev, window, alibi, block_tables, seq_lens_k, block_size, max_blocks, num_blocks);
}

// Backward of cb_flash_attn_fwd for self attention (seqlen_q == seqlen_k).  q / out / dout / dq [T, hq, D], k / v / dk /
// dv [T, hkv, D], lse [T, hq] fp32 from the forward.  Workspaces: delta [T, hq] fp32 and dq_acc [T, hq, D] fp32 (this
// function zeroes dq_acc).  dtype and GQA as the forward; head_dim 128.
// Unlike the forward, the gradients of a sequence are NOT independent of the rows after it: a ragged last key tile or
// query tile loads the next sequence's (or batch entry's) q / k / dout rows, and although their P and dS are forced to
// 0, 0 * NaN or Inf in the dV / dK / dQ MMAs is NaN.  Non-finite values in one packed sequence can therefore corrupt
// the gradients of the sequence before it.
int cb_flash_attn_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const float* lse,
                      void* dq, void* dk, void* dv, float* delta, float* dq_acc, int batch, int seqlen, int hq, int hkv,
                      int head_dim, int causal, float scale, int dtype, const int* cu_seqlens, long long total_tokens,
                      cudaStream_t stream) {
  if (!bwd_args_ok(hq, hkv, head_dim, dtype)) return (int)cudaErrorInvalidValue;
  // cu_seqlens != null: packed batch of `total_tokens` rows (seqlen ignored); else `batch` sequences of `seqlen`
  if (batch <= 0 || (cu_seqlens ? total_tokens <= 0 : seqlen <= 0)) return 0;
  const long long rows = (cu_seqlens ? total_tokens : (long long)batch * seqlen) * hq;
  const long long n = rows * head_dim;
  cudaError_t e = cudaMemsetAsync(dq_acc, 0, (size_t)n * sizeof(float), stream);
  if (e != cudaSuccess) return (int)e;
  int rc = launch_flash_delta(out, dout, delta, rows, head_dim, dtype, stream);
  if (rc) return rc;
  rc = launch_flash_bwd<128>(q, k, v, dout, lse, delta, dq_acc, dk, dv, batch, seqlen, hq, hkv, causal, scale, dtype,
                             stream, cu_seqlens, total_tokens);
  if (rc) return rc;
  const unsigned blocks = (unsigned)((n / 8 + 255) / 256);
  if (dtype == CB_BF16) flash_bwd_cast_dq_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(dq_acc, (__nv_bfloat16*)dq, n);
  else flash_bwd_cast_dq_kernel<__half><<<blocks, 256, 0, stream>>>(dq_acc, (__half*)dq, n);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Blockwise attention for fused ring (context-parallel) attention.  One launch = the queries of this rank against ONE
// key/value block that may live in a PEER's memory (k / v are then peer-mapped symmetric-buffer addresses: the TMA
// loads of the main loop pull the tiles over NVLink, GQA heads only, no staging copy).
//   forward : cb_flash_attn_fwd in block mode.  The online-softmax state (o_state fp32, lse) is carried from launch to
//             launch inside the kernel (`has_prev`), which replaces the reference's per-hop `_rescale_out_lse` pass
//             (`layer/attn.py:376-403`);
//   backward: dQ accumulates in the local fp32 `dq_acc` (not zeroed here), dK / dV are reduced straight into the block
//             owner's fp32 accumulators (`dk_acc` / `dv_acc`, peer pointers) - the reference circulates fp32 dKV
//             buffers around the ring instead (`layer/attn.py:1066-1163`).  `delta` = rowsum(dO o O) is an input.
int cb_flash_attn_block_bwd(const void* q, const void* k, const void* v, const void* dout, const float* lse,
                            const float* delta, float* dq_acc, float* dk_acc, float* dv_acc, int rows, int hq, int hkv,
                            int head_dim, int causal, float scale, int dtype, cudaStream_t stream) {
  if (!bwd_args_ok(hq, hkv, head_dim, dtype) || !dq_acc || !dk_acc || !dv_acc) return (int)cudaErrorInvalidValue;
  if (rows <= 0) return 0;
  return launch_flash_bwd<128>(q, k, v, dout, lse, delta, dq_acc, nullptr, nullptr, 1, rows, hq, hkv, causal, scale, dtype,
                               stream, nullptr, 0, dk_acc, dv_acc);
}

// delta[t, h] = sum_d dO o O for `rows` (token, head) rows of width head_dim
int cb_flash_attn_delta(const void* out, const void* dout, float* delta, long long rows, int head_dim, int dtype,
                        cudaStream_t stream) {
  if (dtype != CB_BF16 && dtype != CB_F16) return (int)cudaErrorInvalidValue;
  if (rows <= 0) return 0;
  return launch_flash_delta(out, dout, delta, rows, head_dim, dtype, stream);
}

}  // extern "C"
