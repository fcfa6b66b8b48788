// Paged-KV inference kernels for sm_90a.
//
// KV cache layout (both K and V, per layer):  [num_blocks, block_size, kv_heads, head_dim]  (token-major inside a block,
// 16-byte vectors along head_dim; one (block, head) tile is a strided 2-D box, i.e. directly TMA-addressable).
//
//   cb_kv_cache_write        : scatter this step's K,V rows [tokens, kv_heads, D] into their paged slots (prefill: all
//                              prompt tokens via cu_seqlens; decode: one token per sequence); a 16-bit cache stores the
//                              rows as they are, an fp8 cache (uint8 bytes) stores them rounded to e5m2
//   cb_paged_decode_attention: split-KV flash-decoding: grid (seq, group of <= 8 kv heads, split); one WARP serves a
//                              kv head (its whole GQA group, so K/V are read once per group) and the warps of a CTA
//                              stream adjacent head slices of the same token rows; fp32 online softmax; second pass
//                              merges splits; an e5m2 cache is decoded exactly to the query dtype after the load, so
//                              the result is bitwise that of the 16-bit cache holding the decoded values.  Head_dim
//                              64 / 128 run on tensor cores, head_dim 256 on CUDA cores.  At head_dim 64 / 128 the
//                              same pass takes q_len <= 16 query tokens per sequence (speculative verification): the
//                              MMA rows are (query token, q head) pairs, so up to 16 / G tokens cost one decode pass
//                              over K/V; each token sees the cache up to its own position, and without a window each
//                              output row is bitwise the single-token result for that token alone
//   cb_convert_fp8           : fp16/bf16/fp32 <-> fp8 e5m2 storage
//
// Capability parity: reference inference_ops_cuda (extensions/csrc/kernel/cuda/{flash_decoding_attention,
// decode_kv_cache_memcpy,context_kv_cache_memcpy,fused_rotary_emb_and_cache,get_cos_and_sin,convert_fp8}_kernel.cu,
// N12-N19) and the Triton twins (kernel/triton/{flash_decoding,kvcache_copy,no_pad_rotary_embedding}.py).
// Decode attention is HBM-bound (every K/V byte is read once): the design goal is full-sector 16-byte loads, many of them
// in flight per SM, and enough CTAs (seqs x kv_heads x splits >= 2 waves of 2 x 132 on an H100) rather than tensor cores.
#include "common.cuh"

namespace {

constexpr int DEC_THREADS = 256;   // at most 8 (kv head, query-head set) units per CTA
constexpr int MAX_GROUP = 8;   // q heads per kv head handled by one CTA

template <typename T> CB_DEVICE float kv_to_f32(T v) { return to_f32<T>(v); }

// 16-byte asynchronous global -> shared copy; src_bytes < 16 zero-fills the rest (0 = pure zero fill)
CB_DEVICE void cp_async_16(void* smem_dst, const void* gmem_src, uint32_t src_bytes) {
  const uint32_t dst = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(gmem_src), "r"(src_bytes) : "memory");
}
CB_DEVICE float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
CB_DEVICE void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> CB_DEVICE void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// fp8 KV cache: a uint8 cache holds e5m2 bytes, written with round-to-nearest-even (as cb_convert_fp8 and
// torch.float8_e5m2 do).  Every e5m2 value is exactly an fp16, bf16 and fp32 value, so decoding is exact.
template <typename T> CB_DEVICE uint2 e5m2_pack8(const uint4 raw) {   // 8 values of T -> 8 e5m2 bytes
  Vec16<T> x;
  x.raw = raw;
  uint32_t w[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(x.get(4 * j), x.get(4 * j + 1)), __NV_SATFINITE, __NV_E5M2);
    const uint32_t hi =
        __nv_cvt_float2_to_fp8x2(make_float2(x.get(4 * j + 2), x.get(4 * j + 3)), __NV_SATFINITE, __NV_E5M2);
    w[j] = lo | (hi << 16);
  }
  return make_uint2(w[0], w[1]);
}
template <typename T> CB_DEVICE uint32_t e5m2x2_decode(uint32_t pair);   // 2 e5m2 bytes (low half) -> 2 values of T
template <> CB_DEVICE uint32_t e5m2x2_decode<__half>(uint32_t pair) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)pair, __NV_E5M2);
  return (uint32_t)h.x | ((uint32_t)h.y << 16);
}
template <> CB_DEVICE uint32_t e5m2x2_decode<__nv_bfloat16>(uint32_t pair) {
  const float2 f = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)pair, __NV_E5M2)));
  __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
  return *reinterpret_cast<uint32_t*>(&b);
}
template <typename T> CB_DEVICE void e5m2_unpack16(const uint4 in, uint4 (&out)[2]) {   // 16 e5m2 bytes -> 16 of T
  const uint32_t w[4] = {in.x, in.y, in.z, in.w};
  uint32_t r[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    r[2 * j] = e5m2x2_decode<T>(w[j] & 0xffffu);
    r[2 * j + 1] = e5m2x2_decode<T>(w[j] >> 16);
  }
  out[0] = make_uint4(r[0], r[1], r[2], r[3]);
  out[1] = make_uint4(r[4], r[5], r[6], r[7]);
}

template <typename T, typename TC>
__global__ void __launch_bounds__(256) kv_cache_write_kernel(const T* __restrict__ k, const T* __restrict__ v,
                                                             TC* __restrict__ k_cache, TC* __restrict__ v_cache,
                                                             const int* __restrict__ block_tables,
                                                             const int* __restrict__ token_seq,   // [tokens] seq id
                                                             const int* __restrict__ token_pos,   // [tokens] position
                                                             int tokens, int kv_heads, int D, int block_size,
                                                             int max_blocks_per_seq, int64_t k_stride,
                                                             int64_t v_stride) {
  const int t = blockIdx.x;
  if (t >= tokens) return;
  const int seq = token_seq[t], pos = token_pos[t];
  const int blk = block_tables[seq * max_blocks_per_seq + pos / block_size];
  const int slot = pos % block_size;
  const int64_t dst = ((int64_t)blk * block_size + slot) * kv_heads * D;
  const int n = kv_heads * D;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    k_cache[dst + i] = (TC)k[(int64_t)t * k_stride + i];
    v_cache[dst + i] = (TC)v[(int64_t)t * v_stride + i];
  }
}

// 16-byte vectorised variants (the hot ones): one thread moves one 16-byte vector, grid = all vectors of the step, so a
// prefill of thousands of tokens is a single HBM-rate streaming kernel instead of one small CTA per token.  An e5m2
// cache (TC = __nv_fp8_e5m2) takes the same 16 input bytes per thread and stores 8.
template <typename T, typename TC>
__global__ void __launch_bounds__(256) kv_cache_write_vec_kernel(const T* __restrict__ k, const T* __restrict__ v,
                                                                 TC* __restrict__ k_cache, TC* __restrict__ v_cache,
                                                                 const int* __restrict__ block_tables,
                                                                 const int* __restrict__ token_seq,
                                                                 const int* __restrict__ token_pos, int tokens,
                                                                 int vec_per_tok, int block_size, int max_blocks_per_seq,
                                                                 int64_t k_stride, int64_t v_stride) {
  // vec_per_tok = kv_heads * D / 8 (16-bit elements); work items = tokens * 2 (K, V) * vec_per_tok
  const int64_t total = (int64_t)tokens * 2 * vec_per_tok;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(w / (2 * vec_per_tok));
    const int r = (int)(w - (int64_t)t * 2 * vec_per_tok);
    const bool is_v = r >= vec_per_tok;
    const int i = is_v ? r - vec_per_tok : r;
    const int seq = __ldg(token_seq + t), pos = __ldg(token_pos + t);
    const int blk = __ldg(block_tables + seq * max_blocks_per_seq + pos / block_size);
    const int64_t dst = ((int64_t)blk * block_size + pos % block_size) * vec_per_tok + i;       // in 8-element units
    const uint4 val = is_v ? __ldg(reinterpret_cast<const uint4*>(v + (int64_t)t * v_stride) + i)
                           : __ldg(reinterpret_cast<const uint4*>(k + (int64_t)t * k_stride) + i);
    if constexpr (sizeof(TC) == 1) reinterpret_cast<uint2*>(is_v ? v_cache : k_cache)[dst] = e5m2_pack8<T>(val);
    else reinterpret_cast<uint4*>(is_v ? v_cache : k_cache)[dst] = val;
  }
}

// One CTA: sequence `seq`, kv head `kvh`, KV partition `split`.  q: [num_seqs, Hq, D].
// partial outputs: o_part [num_seqs, Hq, splits, D] fp32, ml_part [num_seqs, Hq, splits, 2] (max, sumexp)
//
// Work mapping (the kernel is HBM-bound: every K/V byte is read once, so the job is to keep many full-sector loads in
// flight per SM and to spend few instructions per byte):
//   * a K or V row of one (token, kv head) is D contiguous elements; LPT = D/16 adjacent lanes cover one row with two
//     16-byte loads each, so a warp reads 32/LPT whole rows per pass (fully used 32-byte sectors, 128-byte lines);
//   * the rows travel through a per-warp cp.async ring in shared memory (DEC_STAGES stages of DEC_U passes = 4 KB each):
//     3 stages = 12 KB per warp, ~96 KB per SM stay in flight while one stage is consumed - enough to cover the HBM
//     latency at full bandwidth, independent of the register budget (the first two versions kept the rows in
//     registers: 8 warps / SM at 255 registers, 43 % issue-active, 2.4 TB/s under ncu - load and FMA phases of a warp
//     alternated, then only 32 KB per SM in flight); no block-wide barrier in the main loop;
//   * the query rows live in registers (GH = 4 query heads per warp, the lane's 16 dims of each); a GQA group wider
//     than 4 takes two warps of the CTA (the second read of a K/V row by the sibling warp is an L1/L2 hit);
//   * every lane group keeps its OWN online-softmax state (m, l, o) for the tokens it sees - no cross-lane traffic in
//     the loop except the log2(LPT) shuffles that finish a dot product; the 32/LPT states of a warp are merged once at
//     the end and written as this (head set, partition)'s partial result - no shared-memory reduction, no barrier.
constexpr int DEC_U = 2;    // passes of the warp per pipeline stage
constexpr int DEC_STAGES = 4;   // shared-memory ring depth per warp (DEC_STAGES - 1 stages in flight)
constexpr int DEC_GH = 4;   // query heads per warp

template <typename T, typename TC, int D>
__global__ void __launch_bounds__(DEC_THREADS, 1) paged_decode_kernel(
    const T* __restrict__ q, const TC* __restrict__ k_cache, const TC* __restrict__ v_cache,
    const int* __restrict__ block_tables, const int* __restrict__ seq_lens, float* __restrict__ o_part,
    float* __restrict__ ml_part, int Hq, int Hkv, int block_size, int max_blocks_per_seq, int splits, int part_len,
    float scale, const float* __restrict__ alibi_slopes, int64_t q_stride, int window) {
  static_assert(sizeof(TC) == 2 || sizeof(TC) == 1, "16-bit or e5m2 cache");
  constexpr int EPL = 16;                       // elements of a row owned by a lane
  // 16-byte vectors per lane and row: two of 16-bit elements, or one of e5m2 bytes (decoded to T after the load).  An
  // e5m2 ring has twice the stages of half the size: the same shared memory and about the same bytes in flight.
  constexpr int HV = sizeof(TC);
  constexpr int LPT = D / EPL;                  // lanes per token row: 4 / 8 / 16
  constexpr int TPW = 32 / LPT;                 // token rows per warp pass
  constexpr int GH = DEC_GH, U = DEC_U;
  constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
  // CTA = (sequence, group of kv heads, KV partition); warp = one (kv head, set of <= 4 query heads) unit walking ALL
  // tokens of the partition.  The warps of a CTA read ADJACENT 256-byte head slices of the same token rows at the same
  // time, so the CTA streams contiguous [tokens x heads x D] spans of the cache (with one CTA per kv head the 2 KB
  // stride between a head's rows cost ~60 % of the DRAM bandwidth: 2.4 TB/s whatever the number of bytes in flight).
  const int seq = blockIdx.x, split = blockIdx.z;
  const int G = Hq / Hkv;
  const int nsets = (G + GH - 1) / GH;          // sets of <= 4 query heads per kv head
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int unit = blockIdx.y * (blockDim.x >> 5) + warp;
  const int kvh = unit / nsets, set = unit - kvh * nsets;
  if (kvh >= Hkv) return;                       // (no block-wide barrier anywhere in this kernel)
  const int len = seq_lens[seq];
  // sliding-window attention (Mistral): only the last `window` cached tokens are visible - partitions that lie before
  // the window start contribute nothing (m = -inf, l = 0) and are skipped by the merge
  const int window_start = window > 0 ? max(0, len - window) : 0;
  const int t0 = max(split * part_len, window_start), t1 = min(len, split * part_len + part_len);
  const int g0 = set * GH;
  const int ng = min(GH, G - g0);
  const int grp = lane / LPT, sub = lane - grp * LPT;

  float qr[GH][EPL];
#pragma unroll
  for (int g = 0; g < GH; ++g) {
    const T* qp = q + (int64_t)seq * q_stride + (int64_t)(kvh * G + g0 + (g < ng ? g : 0)) * D + sub * EPL;
#pragma unroll
    for (int e = 0; e < EPL; ++e) qr[g][e] = g < ng ? to_f32<T>(qp[e]) * (scale * LOG2E) : 0.f;   // scores in the exp2 domain
  }
  float slope[GH];
#pragma unroll
  for (int g = 0; g < GH; ++g) slope[g] = (alibi_slopes && g < ng) ? alibi_slopes[kvh * G + g0 + g] * LOG2E : 0.f;
  const bool has_alibi = alibi_slopes != nullptr;
  float m[GH], l[GH], o[GH][EPL];
#pragma unroll
  for (int g = 0; g < GH; ++g) {
    m[g] = -INFINITY; l[g] = 0.f;
#pragma unroll
    for (int e = 0; e < EPL; ++e) o[g][e] = 0.f;
  }
  const int* bt = block_tables + seq * max_blocks_per_seq;
  const int bs_shift = (block_size & (block_size - 1)) == 0 ? 31 - __clz(block_size) : -1;   // power-of-two blocks: no division
  // K/V travel through a per-warp ring of DEC_STAGES shared-memory stages filled with cp.async (16 bytes per lane and
  // vector; a stage = U passes of the warp = U * TPW token rows, K and V): the bytes in flight are bounded by shared
  // memory, not by registers, so DEC_STAGES - 1 stages (6 KB) per warp stay outstanding while one is consumed.  Every
  // lane reads back exactly the vectors it requested itself (slot = [stage][k|v][pass][half][lane]), so no barrier is
  // needed beyond cp.async.wait_group, and the 16-byte slots of a warp are consecutive (conflict-free LDS.128).
  extern __shared__ __align__(16) unsigned char dec_smem[];
  constexpr int NST = DEC_STAGES * 2 / HV;
  constexpr int STAGE_VECS = 2 * U * HV * 32;                     // uint4 slots per stage: (K|V) x pass x half x lane
  uint4* ring = reinterpret_cast<uint4*>(dec_smem) + (size_t)warp * NST * STAGE_VECS;
  auto issue_stage = [&](int base, int stage) {
    uint4* st = ring + stage * STAGE_VECS;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int t = base + u * TPW + grp;
      const bool ok = t < t1;
      const int tt = ok ? t : t0;                                 // any valid row: src-size 0 zero-fills instead
      const int blk = bt[bs_shift >= 0 ? (tt >> bs_shift) : (tt / block_size)];
      const int slot = bs_shift >= 0 ? (tt & (block_size - 1)) : (tt % block_size);
      const int64_t row = (((int64_t)blk * block_size + slot) * Hkv + kvh) * D + sub * EPL;
      const uint32_t nbytes = ok ? 16u : 0u;
#pragma unroll
      for (int h = 0; h < HV; ++h) {
        cp_async_16(st + ((0 * U + u) * HV + h) * 32 + lane, k_cache + row + h * 8, nbytes);
        cp_async_16(st + ((1 * U + u) * HV + h) * 32 + lane, v_cache + row + h * 8, nbytes);
      }
    }
  };
  // the lane's 16 elements of a K (kv = 0) or V (kv = 1) row of pass u, as two vectors of T
  auto row_vecs = [&](const uint4* st, int kv, int u, Vec16<T>& a, Vec16<T>& b) {
    if constexpr (HV == 1) {
      uint4 x[2];
      e5m2_unpack16<T>(st[(kv * U + u) * 32 + lane], x);
      a.raw = x[0];
      b.raw = x[1];
    } else {
      a.raw = st[((kv * U + u) * 2 + 0) * 32 + lane];
      b.raw = st[((kv * U + u) * 2 + 1) * 32 + lane];
    }
  };
  auto consume = [&](int base, int stage) {
    const uint4* st = ring + stage * STAGE_VECS;
    float sc[U][GH];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      Vec16<T> k0, k1;
      row_vecs(st, 0, u, k0, k1);
      const int t = base + u * TPW + grp;
#pragma unroll
      for (int g = 0; g < GH; ++g) {
        float acc = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc += qr[g][e] * k0.get(e);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc += qr[g][8 + e] * k1.get(e);
#pragma unroll
        for (int off = LPT / 2; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
        if (has_alibi) acc += slope[g] * (float)(t - (len - 1));
        sc[u][g] = (t < t1) ? acc : -INFINITY;
      }
    }
    float pr[U][GH];
#pragma unroll
    for (int g = 0; g < GH; ++g) {
      float nm = m[g];
#pragma unroll
      for (int u = 0; u < U; ++u) nm = fmaxf(nm, sc[u][g]);
      if (__any_sync(0xffffffffu, nm > m[g])) {                   // the running max moved for some row group: rescale
        const float corr = (nm == -INFINITY) ? 1.f : ex2_approx(m[g] - nm);
        l[g] *= corr;
#pragma unroll
        for (int e = 0; e < EPL; ++e) o[g][e] *= corr;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        pr[u][g] = (sc[u][g] == -INFINITY) ? 0.f : ex2_approx(sc[u][g] - nm);
        l[g] += pr[u][g];
      }
      m[g] = nm;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      Vec16<T> v0, v1;
      row_vecs(st, 1, u, v0, v1);
#pragma unroll
      for (int g = 0; g < GH; ++g) {
#pragma unroll
        for (int e = 0; e < 8; ++e) o[g][e] += pr[u][g] * v0.get(e);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[g][8 + e] += pr[u][g] * v1.get(e);
      }
    }
  };
  {
    const int step = TPW * U;
    const int first = t0;
    // prologue: NST - 1 stages in flight (empty groups keep the group count uniform at the tail)
#pragma unroll
    for (int s = 0; s < NST - 1; ++s) {
      if (first + s * step < t1) issue_stage(first + s * step, s);
      cp_async_commit();
    }
    int it = 0;
    for (int base = first; base < t1; base += step, ++it) {
      const int ahead = base + (NST - 1) * step;
      if (ahead < t1) issue_stage(ahead, (it + NST - 1) % NST);
      cp_async_commit();
      cp_async_wait<NST - 1>();                                   // the group of stage `it` has landed
      consume(base, it % NST);
    }
    cp_async_wait<0>();
  }
  // merge the TPW lane-group states of the warp (butterfly over the group index)
#pragma unroll
  for (int off = LPT; off < 32; off <<= 1) {
#pragma unroll
    for (int g = 0; g < GH; ++g) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[g], off);
      const float lo = __shfl_xor_sync(0xffffffffu, l[g], off);
      const float nm = fmaxf(m[g], mo);
      const float c1 = (m[g] == -INFINITY) ? 0.f : ex2_approx(m[g] - nm);
      const float c2 = (mo == -INFINITY) ? 0.f : ex2_approx(mo - nm);
      l[g] = l[g] * c1 + lo * c2;
#pragma unroll
      for (int e = 0; e < EPL; ++e) o[g][e] = o[g][e] * c1 + __shfl_xor_sync(0xffffffffu, o[g][e], off) * c2;
      m[g] = nm;
    }
  }
  // every lane group now holds the merged state; group 0 writes this unit's partial result
  if (grp == 0) {
#pragma unroll
    for (int g = 0; g < GH; ++g) {
      if (g < ng) {
        const int64_t oi = (((int64_t)seq * Hq + kvh * G + g0 + g) * splits + split);
        float4* dst = reinterpret_cast<float4*>(o_part + oi * D + sub * EPL);
#pragma unroll
        for (int e = 0; e < EPL; e += 4) dst[e >> 2] = make_float4(o[g][e], o[g][e + 1], o[g][e + 2], o[g][e + 3]);
        if (sub == 0) { ml_part[oi * 2] = m[g] * LN2; ml_part[oi * 2 + 1] = l[g]; }   // max back in natural-log units
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------------------------
// Tensor-core formulation of the same split-KV decode step (head_dim 64 / 128; the kernel above serves head_dim 256).
//
// The CUDA-core kernel above executes ~89 warp-instructions per (token, kv head) - two FMAs per cached element and q
// head - which is as much issue time as the HBM transfer takes (ncu: 93 M warp-instructions, 45 % issue-active,
// 2.2-2.4 TB/s).  Here the GQA group of a kv head (<= 8 q heads, padded to the 16 rows of an MMA) is the M dimension of
// `mma.sync.m16n8k16`:  S[heads x 16 tokens] = Q K^T  and  O[heads x D] += P V  per 16-token tile, i.e. 32 MMAs instead of
// ~4000 FMAs per tile and lane.
//   * warp = (sequence, kv head, partition) unit, as above; Q fragments (A operand) live in registers;
//   * a tile of 16 token rows of K and of V (16 x D 16-bit values each) is fetched with cp.async into a per-warp ring
//     (DEC_MMA_STAGES deep); a row's 16-byte chunks are stored XOR-swizzled by (token mod 8), so the ldmatrix reads - K
//     plain (B operand of Q K^T), V transposed (B operand of P V) - are bank-conflict free;
//   * softmax state per head row is replicated over the four lanes of a quad; the probabilities go straight from the
//     accumulator layout of S to the A-operand layout of P V (no shared-memory round trip); the output accumulator is
//     rescaled only when a row max moved;
//   * partial results use the same (o_part, ml_part) format, so the reduce kernel is shared.
// An e5m2 cache (TC = __nv_fp8_e5m2) travels through the ring as bytes (half a 16-bit stage each, so 5 stages keep the
// 16-bit ring's bytes in flight); the warp decodes the landed stage into one swizzled 16-bit K,V tile pair before the
// ldmatrix reads, so the MMAs and everything after them are those of the 16-bit kernel.
constexpr int DEC_MMA_TOKENS = 16;
constexpr int DEC_MMA_STAGES = 3;

template <typename TC> constexpr int dec_mma_stages() { return sizeof(TC) == 1 ? 5 : DEC_MMA_STAGES; }
template <typename TC, int D> constexpr int dec_mma_smem_per_warp() {
  return dec_mma_stages<TC>() * 2 * DEC_MMA_TOKENS * D * (int)sizeof(TC) + (sizeof(TC) == 1 ? 2 * DEC_MMA_TOKENS * D * 2 : 0);
}

CB_DEVICE void ldmatrix_x4(uint32_t (&r)[4], const void* smem_row) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
CB_DEVICE void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
template <typename T> CB_DEVICE void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <> CB_DEVICE void mma_16816<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> CB_DEVICE void mma_16816<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <typename T> CB_DEVICE uint32_t pack2(float lo, float hi);
template <> CB_DEVICE uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <> CB_DEVICE uint32_t pack2<__half>(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Multi-query form (MQ, speculative verification): q_len query tokens per sequence, q / out rows seq * q_len + j.  The
// MMA rows are the flattened (query token j, q head g) pairs r = j * G + g, all 16 of them used; a warp is one (kv head,
// 16-row slice) unit, and when q_len * G > 16 the sibling warps of a kv head stream (and, for e5m2, decode) the same K/V
// tiles, meant to hit L1 / L2 on the second read.  Query j sees the len_j = len - (q_len - 1 - j) first positions (the last `window` of them); each
// row masks its own range, the tiles keep their bases at split * part_len and run to the warp's longest row, and a
// masked position adds p = 0 - so without a window each row is bitwise the decode kernel's result for that row alone.
// A window starts the tile grid at the warp's first row's window start, so windowed rows match only to rounding.
// The decode kernel is the MQ = false instantiation with q_len = 1 (the upper 8 MMA rows stay zero padding).
template <typename T, typename TC, int D, bool MQ>
CB_DEVICE void paged_mma_attend(
    const T* __restrict__ q, const TC* __restrict__ k_cache, const TC* __restrict__ v_cache,
    const int* __restrict__ block_tables, const int* __restrict__ seq_lens, float* __restrict__ o_part,
    float* __restrict__ ml_part, int Hq, int Hkv, int block_size, int max_blocks_per_seq, int splits, int part_len,
    float scale, const float* __restrict__ alibi_slopes, int64_t q_stride, int window, int q_len) {
  static_assert(sizeof(TC) == 2 || sizeof(TC) == 1, "16-bit or e5m2 cache");
  constexpr bool F8 = sizeof(TC) == 1;
  constexpr int NT = DEC_MMA_TOKENS, NST = dec_mma_stages<TC>();
  constexpr int KS = D / 16;                    // k-steps of Q K^T
  constexpr int NO = D / 8;                     // 8-wide column tiles of the output
  constexpr int CPR = D * (int)sizeof(TC) / 16; // 16-byte chunks per cached token row
  constexpr int ROW_BYTES = D * 2;              // a token row of a 16-bit tile
  constexpr int TILE_BYTES = NT * ROW_BYTES;    // one 16-bit operand (K or V) tile
  constexpr int STAGE_BYTES = 2 * NT * D * (int)sizeof(TC);   // K and V of one stage as cached
  constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
  const int seq = blockIdx.x, split = blockIdx.z;
  const int G = Hq / Hkv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nrows = q_len * G;                  // MMA rows of a kv head: (query token, q head) pairs
  const int nslices = MQ ? (nrows + 15) >> 4 : 1;
  const int unit = blockIdx.y * (blockDim.x >> 5) + warp;
  const int kvh = unit / nslices, r0 = (unit - kvh * nslices) * 16;   // kv head, first MMA row of the warp's slice
  if (kvh >= Hkv) return;                       // (no block-wide barrier in this kernel)
  const int len = seq_lens[seq];
  // positions [lo, hi) of this partition that query token j sees
  auto visible = [&](int j, int& lo, int& hi) {
    const int len_j = len - (q_len - 1 - j);
    const int window_start = window > 0 ? max(0, len_j - window) : 0;
    lo = max(split * part_len, window_start);
    hi = min(len_j, split * part_len + part_len);
  };
  int t0, t1, unused;                           // the warp's tile range: first row's start to last row's end
  visible(MQ ? r0 / G : 0, t0, unused);
  visible(MQ ? (min(nrows, r0 + 16) - 1) / G : 0, unused, t1);
  const int row = lane >> 2, quad = lane & 3;   // accumulator layout: head row, column pair inside an 8-wide tile
  const bool row_ok = row < G;                  // rows G..15 of the MMA are padding
  const float scale2 = scale * LOG2E;           // scores in the exp2 domain
  const float slope2 = (alibi_slopes != nullptr && row_ok) ? alibi_slopes[kvh * G + row] * LOG2E : 0.f;
  const bool has_alibi = alibi_slopes != nullptr;
  // MQ: this lane's two MMA rows, r0 + row (h = 0, accumulator regs 0 / 1) and r0 + row + 8 (h = 1, regs 2 / 3)
  bool rok[2];
  int rq[2], rhead[2], rlen[2], rlo[2], rhi[2];
  float rslope[2];
  if constexpr (MQ) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + row + 8 * h;
      rok[h] = r < nrows;
      rq[h] = rok[h] ? r / G : 0;
      rhead[h] = kvh * G + (rok[h] ? r - rq[h] * G : 0);
      rlen[h] = len - (q_len - 1 - rq[h]);
      visible(rq[h], rlo[h], rhi[h]);
      if (!rok[h]) rlo[h] = rhi[h] = 0;         // padding row: every position masked
      rslope[h] = (alibi_slopes != nullptr && rok[h]) ? alibi_slopes[rhead[h]] * LOG2E : 0.f;
    }
  }

  // ---- Q fragments: A operand [16 rows x 16 d] per k-step; decode: a1 / a3 are head rows 8..15 = zero (G <= 8)
  uint32_t qa[KS][4];
  if constexpr (MQ) {
    const T* qr0 = q + (int64_t)(seq * q_len + rq[0]) * q_stride + (int64_t)rhead[0] * D;
    const T* qr1 = q + (int64_t)(seq * q_len + rq[1]) * q_stride + (int64_t)rhead[1] * D;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const uint32_t lo0 = *reinterpret_cast<const uint32_t*>(qr0 + ks * 16 + quad * 2);
      const uint32_t hi0 = *reinterpret_cast<const uint32_t*>(qr0 + ks * 16 + 8 + quad * 2);
      const uint32_t lo1 = *reinterpret_cast<const uint32_t*>(qr1 + ks * 16 + quad * 2);
      const uint32_t hi1 = *reinterpret_cast<const uint32_t*>(qr1 + ks * 16 + 8 + quad * 2);
      qa[ks][0] = rok[0] ? lo0 : 0u; qa[ks][1] = rok[1] ? lo1 : 0u;
      qa[ks][2] = rok[0] ? hi0 : 0u; qa[ks][3] = rok[1] ? hi1 : 0u;
    }
  } else {
    const T* qrow = q + (int64_t)seq * q_stride + (int64_t)(kvh * G + (row_ok ? row : 0)) * D;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const uint32_t lo = *reinterpret_cast<const uint32_t*>(qrow + ks * 16 + quad * 2);
      const uint32_t hi = *reinterpret_cast<const uint32_t*>(qrow + ks * 16 + 8 + quad * 2);
      qa[ks][0] = row_ok ? lo : 0u; qa[ks][1] = 0u; qa[ks][2] = row_ok ? hi : 0u; qa[ks][3] = 0u;
    }
  }
  float o[NO][4];
#pragma unroll
  for (int j = 0; j < NO; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
  float m_run = -INFINITY, l_run = 0.f;         // per head row, replicated over the quad (l: this lane's share)
  float mq_m[2] = {-INFINITY, -INFINITY}, mq_l[2] = {0.f, 0.f};   // MQ: the same for rows h = 0, 1

  extern __shared__ __align__(128) unsigned char dec_smem[];
  unsigned char* ring = dec_smem + (F8 ? (size_t)warp * dec_mma_smem_per_warp<TC, D>() : (size_t)warp * NST * 2 * TILE_BYTES);
  unsigned char* decoded = ring + NST * STAGE_BYTES;         // e5m2: the stage being consumed, as a 16-bit K,V tile
  const int* bt = block_tables + seq * max_blocks_per_seq;
  const int bs_shift = (block_size & (block_size - 1)) == 0 ? 31 - __clz(block_size) : -1;
  auto issue_stage = [&](int base, int stage) {
    unsigned char* kt = ring + (size_t)stage * STAGE_BYTES;
    unsigned char* vt = kt + STAGE_BYTES / 2;
#pragma unroll
    for (int i = 0; i < NT * CPR / 32; ++i) {
      const int cid = lane + 32 * i;
      const int tr = cid / CPR, c = cid - tr * CPR;          // token row inside the tile, 16-byte chunk inside the row
      const int t = base + tr;
      const bool ok = t < t1;
      const int tt = ok ? t : t0;
      const int blk = bt[bs_shift >= 0 ? (tt >> bs_shift) : (tt / block_size)];
      const int slot = bs_shift >= 0 ? (tt & (block_size - 1)) : (tt % block_size);
      const int64_t src = (((int64_t)blk * block_size + slot) * Hkv + kvh) * D + c * (16 / (int)sizeof(TC));
      const int dst = F8 ? tr * D + (c << 4) : tr * ROW_BYTES + ((c ^ (tr & 7)) << 4);   // e5m2 bytes: unswizzled
      const uint32_t nbytes = ok ? 16u : 0u;
      cp_async_16(kt + dst, k_cache + src, nbytes);
      cp_async_16(vt + dst, v_cache + src, nbytes);
    }
  };
  // e5m2 stage -> `decoded`: each lane decodes the chunks it loaded into the 16-bit tiles' swizzled layout
  auto decode_stage = [&](const unsigned char* kt8) {
#pragma unroll
    for (int i = 0; i < NT * CPR / 32; ++i) {
      const int cid = lane + 32 * i;
      const int tr = cid / CPR, c = cid - tr * CPR;
#pragma unroll
      for (int kv = 0; kv < 2; ++kv) {
        uint4 x[2];
        e5m2_unpack16<T>(*reinterpret_cast<const uint4*>(kt8 + kv * (STAGE_BYTES / 2) + tr * D + (c << 4)), x);
        unsigned char* row16 = decoded + kv * TILE_BYTES + tr * ROW_BYTES;
        *reinterpret_cast<uint4*>(row16 + (((2 * c) ^ (tr & 7)) << 4)) = x[0];
        *reinterpret_cast<uint4*>(row16 + (((2 * c + 1) ^ (tr & 7)) << 4)) = x[1];
      }
    }
  };
  auto consume = [&](int base, int stage) {
    const unsigned char* kt = F8 ? decoded : ring + (size_t)stage * STAGE_BYTES;
    const unsigned char* vt = kt + TILE_BYTES;
    // ---- S = Q K^T for 16 tokens (two 8-token column tiles)
    float sacc[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0.f;
      const int tr = nt * 8 + (lane & 7);                    // token row whose address this lane supplies
#pragma unroll
      for (int ks = 0; ks < KS; ks += 2) {
        // matrices: (ks, d 0..7), (ks, d 8..15), (ks + 1, d 0..7), (ks + 1, d 8..15)
        const int c = 2 * ks + (lane >> 3);
        uint32_t b[4];
        ldmatrix_x4(b, kt + tr * ROW_BYTES + ((c ^ (tr & 7)) << 4));
        mma_16816<T>(sacc[nt], qa[ks], b[0], b[1]);
        mma_16816<T>(sacc[nt], qa[ks + 1], b[2], b[3]);
      }
    }
    uint32_t pa[4];                                          // P as the A operand [16 rows x 16 tokens]
    if constexpr (MQ) {
      // ---- online softmax of rows r0 + row + 8 h, each masked to its own [rlo, rhi); the same operations, in the
      // same order, as the decode path below applies to its one row
      float sv[2][4], m_new[2];
      bool moved = false;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int t = base + nt * 8 + quad * 2 + e;
            float x = sacc[nt][2 * h + e] * scale2;
            if (has_alibi) x = fmaf(rslope[h], (float)(t - (rlen[h] - 1)), x);
            x = (t >= rlo[h] && t < rhi[h]) ? x : -INFINITY;
            sv[h][nt * 2 + e] = x;
            mx = fmaxf(mx, x);
          }
        }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        m_new[h] = fmaxf(mq_m[h], mx);
        moved = moved || m_new[h] > mq_m[h];
      }
      if (__any_sync(0xffffffffu, moved)) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float corr = (m_new[h] == -INFINITY) ? 1.f : ex2_approx(mq_m[h] - m_new[h]);
          mq_l[h] *= corr;
#pragma unroll
          for (int j = 0; j < NO; ++j) { o[j][2 * h] *= corr; o[j][2 * h + 1] *= corr; }
        }
      }
      float pv[2][4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mq_m[h] = m_new[h];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          pv[h][i] = (sv[h][i] == -INFINITY) ? 0.f : ex2_approx(sv[h][i] - m_new[h]);
          mq_l[h] += pv[h][i];
        }
      }
      pa[0] = pack2<T>(pv[0][0], pv[0][1]); pa[1] = pack2<T>(pv[1][0], pv[1][1]);
      pa[2] = pack2<T>(pv[0][2], pv[0][3]); pa[3] = pack2<T>(pv[1][2], pv[1][3]);
    } else {
      // ---- online softmax of head row `row` (this lane: tokens nt * 8 + quad * 2 + {0, 1})
      float sv[4];
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int t = base + nt * 8 + quad * 2 + e;
          float x = sacc[nt][e] * scale2;
          if (has_alibi) x = fmaf(slope2, (float)(t - (len - 1)), x);
          x = (t < t1) ? x : -INFINITY;
          sv[nt * 2 + e] = x;
          mx = fmaxf(mx, x);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run, mx);
      if (__any_sync(0xffffffffu, m_new > m_run)) {
        const float corr = (m_new == -INFINITY) ? 1.f : ex2_approx(m_run - m_new);
        l_run *= corr;
#pragma unroll
        for (int j = 0; j < NO; ++j) { o[j][0] *= corr; o[j][1] *= corr; }
      }
      m_run = m_new;
      float pv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        pv[i] = (sv[i] == -INFINITY) ? 0.f : ex2_approx(sv[i] - m_new);
        l_run += pv[i];
      }
      // a0 = tokens 0..7 of this row, a2 = tokens 8..15; rows 8..15 are zero
      pa[0] = row_ok ? pack2<T>(pv[0], pv[1]) : 0u; pa[1] = 0u;
      pa[2] = row_ok ? pack2<T>(pv[2], pv[3]) : 0u; pa[3] = 0u;
    }
    // ---- O += P V: V^T fragments through ldmatrix.trans
    {
      const int tr = (lane & 7) + ((lane >> 3) & 1) * 8;     // matrices: (tok 0..7, j), (tok 8..15, j), (0..7, j+1), (8..15, j+1)
#pragma unroll
      for (int j = 0; j < NO; j += 2) {
        const int c = j + (lane >> 4);
        uint32_t b[4];
        ldmatrix_x4_trans(b, vt + tr * ROW_BYTES + ((c ^ (tr & 7)) << 4));
        mma_16816<T>(o[j], pa, b[0], b[1]);
        mma_16816<T>(o[j + 1], pa, b[2], b[3]);
      }
    }
  };
  {
#pragma unroll
    for (int s = 0; s < NST - 1; ++s) {
      if (t0 + s * NT < t1) issue_stage(t0 + s * NT, s);
      cp_async_commit();
    }
    int it = 0;
    for (int base = t0; base < t1; base += NT, ++it) {
      const int ahead = base + (NST - 1) * NT;
      if (ahead < t1) issue_stage(ahead, (it + NST - 1) % NST);
      cp_async_commit();
      cp_async_wait<NST - 1>();
      __syncwarp();                                          // the tile was written by all lanes of the warp
      if constexpr (F8) {
        decode_stage(ring + (size_t)(it % NST) * STAGE_BYTES);
        __syncwarp();                                        // the decoded tile was written by all lanes
      }
      consume(base, it % NST);
      __syncwarp();                                          // all lanes done reading before the stage is refilled
    }
    cp_async_wait<0>();
  }
  // ---- this unit's partial result (row sum over the quad first)
  if constexpr (MQ) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mq_l[h] += __shfl_xor_sync(0xffffffffu, mq_l[h], 1);
      mq_l[h] += __shfl_xor_sync(0xffffffffu, mq_l[h], 2);
      if (rok[h]) {
        const int64_t oi = (((int64_t)(seq * q_len + rq[h]) * Hq + rhead[h]) * splits + split);
        float* dst = o_part + oi * D + quad * 2;
#pragma unroll
        for (int j = 0; j < NO; ++j) *reinterpret_cast<float2*>(dst + j * 8) = make_float2(o[j][2 * h], o[j][2 * h + 1]);
        if (quad == 0) { ml_part[oi * 2] = mq_m[h] * LN2; ml_part[oi * 2 + 1] = mq_l[h]; }
      }
    }
    return;
  }
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
  if (row_ok) {
    const int64_t oi = (((int64_t)seq * Hq + kvh * G + row) * splits + split);
    float* dst = o_part + oi * D + quad * 2;
#pragma unroll
    for (int j = 0; j < NO; ++j) *reinterpret_cast<float2*>(dst + j * 8) = make_float2(o[j][0], o[j][1]);
    if (quad == 0) { ml_part[oi * 2] = m_run * LN2; ml_part[oi * 2 + 1] = l_run; }
  }
}

// MQ = false ignores q_len: the decode instantiation is compiled for exactly one query token per sequence.
template <typename T, typename TC, int D, bool MQ>
__global__ void __launch_bounds__(DEC_THREADS, 1) paged_mma_kernel(
    const T* __restrict__ q, const TC* __restrict__ k_cache, const TC* __restrict__ v_cache,
    const int* __restrict__ block_tables, const int* __restrict__ seq_lens, float* __restrict__ o_part,
    float* __restrict__ ml_part, int Hq, int Hkv, int block_size, int max_blocks_per_seq, int splits, int part_len,
    float scale, const float* __restrict__ alibi_slopes, int64_t q_stride, int window, int q_len) {
  paged_mma_attend<T, TC, D, MQ>(q, k_cache, v_cache, block_tables, seq_lens, o_part, ml_part, Hq, Hkv, block_size,
                                 max_blocks_per_seq, splits, part_len, scale, alibi_slopes, q_stride, window,
                                 MQ ? q_len : 1);
}

template <typename T, int D>
__global__ void __launch_bounds__(128) decode_reduce_kernel(const float* __restrict__ o_part,
                                                            const float* __restrict__ ml_part, T* __restrict__ out,
                                                            int Hq, int splits, int64_t out_stride) {
  const int seq = blockIdx.x, h = blockIdx.y;
  const int64_t base = ((int64_t)seq * Hq + h) * splits;
  float gm = -INFINITY;
  for (int s = 0; s < splits; ++s) gm = fmaxf(gm, ml_part[(base + s) * 2]);
  float ls = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float mm = ml_part[(base + s) * 2];
    ls += (mm == -INFINITY) ? 0.f : ml_part[(base + s) * 2 + 1] * __expf(mm - gm);
  }
  const float inv = ls > 0.f ? 1.f / ls : 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) {
      const float mm = ml_part[(base + s) * 2];
      if (mm != -INFINITY) acc += o_part[(base + s) * D + d] * __expf(mm - gm);
    }
    out[(int64_t)seq * out_stride + (int64_t)h * D + d] = from_f32<T>(acc * inv);
  }
}

template <typename TI, typename TO>
__global__ void convert_kernel(const TI* __restrict__ in, TO* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (TO)(float)in[i];
}

// cb_paged_decode_attention's arguments, shared by the launchers below
struct PagedArgs {
  const void *q, *k_cache, *v_cache;
  const int *block_tables, *seq_lens;
  void* out;
  float *o_part, *ml_part;
  int num_seqs, q_len, Hq, Hkv, block_size, max_blocks_per_seq, splits, part_len;
  float scale;
  const float* alibi_slopes;
  int64_t q_stride, out_stride;
  int window;
  cudaStream_t s;
};

// Tensor-core split-KV pass, then the reduce: one warp per (kv head, 16-row slice of its q_len x G rows).
template <typename T, typename TC, int D, bool MQ> void launch_paged_mma(const PagedArgs& a) {
  constexpr int per_warp = dec_mma_smem_per_warp<TC, D>();
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(paged_mma_kernel<T, TC, D, MQ>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (DEC_THREADS / 32) * per_warp);
    attr_done = true;
  }
  const int units = a.Hkv * ((a.q_len * (a.Hq / a.Hkv) + 15) / 16);
  const int warps = units < DEC_THREADS / 32 ? units : DEC_THREADS / 32;
  paged_mma_kernel<T, TC, D, MQ><<<dim3(a.num_seqs, (units + warps - 1) / warps, a.splits), warps * 32,
                                   warps * per_warp, a.s>>>(
      (const T*)a.q, (const TC*)a.k_cache, (const TC*)a.v_cache, a.block_tables, a.seq_lens, a.o_part, a.ml_part, a.Hq,
      a.Hkv, a.block_size, a.max_blocks_per_seq, a.splits, a.part_len, a.scale, a.alibi_slopes, a.q_stride, a.window,
      a.q_len);
  decode_reduce_kernel<T, D><<<dim3(a.num_seqs * a.q_len, a.Hq), 128, 0, a.s>>>(a.o_part, a.ml_part, (T*)a.out, a.Hq,
                                                                               a.splits, a.out_stride);
}

// CUDA-core split-KV pass at head_dim 256 (one query token per sequence), then the reduce: one warp per (kv head,
// set of <= 4 q heads).
template <typename T, typename TC> void launch_paged_cuda_core(const PagedArgs& a) {
  constexpr int ring_bytes = DEC_STAGES * (2 * DEC_U * 2 * 32) * 16;                  // per-warp cp.async ring
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(paged_decode_kernel<T, TC, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (DEC_THREADS / 32) * ring_bytes);
    attr_done = true;
  }
  const int units = a.Hkv * ((a.Hq / a.Hkv + DEC_GH - 1) / DEC_GH);
  const int warps = units < DEC_THREADS / 32 ? units : DEC_THREADS / 32;
  paged_decode_kernel<T, TC, 256><<<dim3(a.num_seqs, (units + warps - 1) / warps, a.splits), warps * 32,
                                    warps * ring_bytes, a.s>>>(
      (const T*)a.q, (const TC*)a.k_cache, (const TC*)a.v_cache, a.block_tables, a.seq_lens, a.o_part, a.ml_part, a.Hq,
      a.Hkv, a.block_size, a.max_blocks_per_seq, a.splits, a.part_len, a.scale, a.alibi_slopes, a.q_stride, a.window);
  decode_reduce_kernel<T, 256><<<dim3(a.num_seqs, a.Hq), 128, 0, a.s>>>(a.o_part, a.ml_part, (T*)a.out, a.Hq, a.splits,
                                                                        a.out_stride);
}

template <typename T, typename TC> void launch_paged(const PagedArgs& a, int D) {
  if (D == 256) launch_paged_cuda_core<T, TC>(a);
  else if (D == 128) a.q_len == 1 ? launch_paged_mma<T, TC, 128, false>(a) : launch_paged_mma<T, TC, 128, true>(a);
  else a.q_len == 1 ? launch_paged_mma<T, TC, 64, false>(a) : launch_paged_mma<T, TC, 64, true>(a);
}

}  // namespace

extern "C" {

// k, v: [tokens, kv_heads, D] (row strides in elements) of `dtype`; the caches hold `cache_dtype`: the same dtype, or
// CB_F8E5M2 (e5m2 bytes, rounded to nearest even).
int cb_kv_cache_write(const void* k, const void* v, void* k_cache, void* v_cache, const int* block_tables,
                      const int* token_seq, const int* token_pos, int tokens, int kv_heads, int D, int block_size,
                      int max_blocks_per_seq, int64_t k_stride, int64_t v_stride, int dtype, int cache_dtype,
                      cudaStream_t s) {
  if (tokens == 0) return 0;
  if (cache_dtype != dtype && cache_dtype != CB_F8E5M2) return (int)cudaErrorInvalidValue;
  const bool f8 = cache_dtype == CB_F8E5M2;
  const int n = kv_heads * D;
  if (n % 8 == 0 && k_stride % 8 == 0 && v_stride % 8 == 0 && ((uintptr_t)k % 16) == 0 && ((uintptr_t)v % 16) == 0 &&
      ((uintptr_t)k_cache % 16) == 0 && ((uintptr_t)v_cache % 16) == 0) {
    const int64_t total = (int64_t)tokens * 2 * (n / 8);
    const int grid = (int)((total + 255) / 256 < 16 * cb_num_sms() ? (total + 255) / 256 : 16 * cb_num_sms());
#define LAUNCH_KV_WRITE_VEC(TC)                                                                                       \
  kv_cache_write_vec_kernel<T, TC><<<grid, 256, 0, s>>>((const T*)k, (const T*)v, (TC*)k_cache, (TC*)v_cache,           \
                                                        block_tables, token_seq, token_pos, tokens, n / 8, block_size, \
                                                        max_blocks_per_seq, k_stride, v_stride)
    CB_DISPATCH_HALF(dtype, T, {
      if (f8) LAUNCH_KV_WRITE_VEC(__nv_fp8_e5m2);
      else LAUNCH_KV_WRITE_VEC(T);
    });
#undef LAUNCH_KV_WRITE_VEC
    return CB_LAUNCH_CHECK();
  }
#define LAUNCH_KV_WRITE(TC)                                                                                           \
  kv_cache_write_kernel<T, TC><<<tokens, 256, 0, s>>>((const T*)k, (const T*)v, (TC*)k_cache, (TC*)v_cache,             \
                                                      block_tables, token_seq, token_pos, tokens, kv_heads, D,         \
                                                      block_size, max_blocks_per_seq, k_stride, v_stride)
  CB_DISPATCH_HALF(dtype, T, {
    if (f8) LAUNCH_KV_WRITE(__nv_fp8_e5m2);
    else LAUNCH_KV_WRITE(T);
  });
#undef LAUNCH_KV_WRITE
  return CB_LAUNCH_CHECK();
}

// Paged attention for q_len query tokens per sequence.  q, out: [num_seqs * q_len, Hq, D] of `dtype`, token-major
// (sequence i's queries are rows i * q_len + j; query j sits at position seq_lens[i] - q_len + j and sees the positions
// before it and itself); caches [nb, bs, Hkv, D] of `cache_dtype` (`dtype` or CB_F8E5M2); o_part fp32
// [num_seqs * q_len, Hq, splits, D], ml_part [.., 2]; splits / part_len as `ops/inference.py` `decode_splits` gives
// them for num_seqs sequences, whatever q_len.  Served: G = Hq / Hkv <= 8 with head_dim 64 / 128 and
// 1 <= q_len <= 16 (tensor cores), or head_dim 256 and q_len = 1 (CUDA cores); anything else launches nothing and
// returns cudaErrorInvalidValue.
int cb_paged_decode_attention(const void* q, const void* k_cache, const void* v_cache, const int* block_tables,
                              const int* seq_lens, void* out, float* o_part, float* ml_part, int num_seqs, int q_len,
                              int Hq, int Hkv, int D, int block_size, int max_blocks_per_seq, int splits, int part_len,
                              float scale, const float* alibi_slopes, int64_t q_stride, int64_t out_stride, int dtype,
                              int cache_dtype, int window, cudaStream_t s) {
  const int max_q_len = (D == 64 || D == 128) ? 16 : D == 256 ? 1 : 0;
  if (Hkv <= 0 || Hq % Hkv != 0 || Hq / Hkv > MAX_GROUP || q_len < 1 || q_len > max_q_len)
    return (int)cudaErrorInvalidValue;
  if (cache_dtype != dtype && cache_dtype != CB_F8E5M2) return (int)cudaErrorInvalidValue;
  if (num_seqs == 0) return 0;
  const PagedArgs a{q, k_cache, v_cache, block_tables, seq_lens, out, o_part, ml_part, num_seqs, q_len, Hq, Hkv,
                    block_size, max_blocks_per_seq, splits, part_len, scale, alibi_slopes, q_stride, out_stride,
                    window, s};
  CB_DISPATCH_HALF(dtype, T, {
    if (cache_dtype == CB_F8E5M2) launch_paged<T, __nv_fp8_e5m2>(a, D);
    else launch_paged<T, T>(a, D);
  });
  return CB_LAUNCH_CHECK();
}

// direction 0: (fp16|bf16|fp32) -> e5m2 ; 1: e5m2 -> (fp16|bf16|fp32)
int cb_convert_fp8(const void* in, void* out, int64_t n, int dtype, int direction, cudaStream_t s) {
  if (n == 0) return 0;
  const int grid = (int)((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256);
  if (direction == 0) {
    if (dtype == CB_BF16) convert_kernel<__nv_bfloat16, __nv_fp8_e5m2><<<grid, 256, 0, s>>>((const __nv_bfloat16*)in, (__nv_fp8_e5m2*)out, n);
    else if (dtype == CB_F16) convert_kernel<__half, __nv_fp8_e5m2><<<grid, 256, 0, s>>>((const __half*)in, (__nv_fp8_e5m2*)out, n);
    else convert_kernel<float, __nv_fp8_e5m2><<<grid, 256, 0, s>>>((const float*)in, (__nv_fp8_e5m2*)out, n);
  } else {
    if (dtype == CB_BF16) convert_kernel<__nv_fp8_e5m2, __nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_fp8_e5m2*)in, (__nv_bfloat16*)out, n);
    else if (dtype == CB_F16) convert_kernel<__nv_fp8_e5m2, __half><<<grid, 256, 0, s>>>((const __nv_fp8_e5m2*)in, (__half*)out, n);
    else convert_kernel<__nv_fp8_e5m2, float><<<grid, 256, 0, s>>>((const __nv_fp8_e5m2*)in, (float*)out, n);
  }
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
