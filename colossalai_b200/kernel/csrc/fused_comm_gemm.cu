// Fused compute + collective kernels for tensor / sequence parallel linears over NVLink peer memory (sm_90a).
//
//   cb_ag_gemm   : Y[T, N]   = all_gather(x_local)[T, K] * B        (col-linear fwd under SP, and dX = AG(dY) * W)
//   cb_gemm_rs   : y_local   = reduce_scatter(A[T, K] * B)          (row-linear fwd under SP, and dX of col-linear)
//   cb_all_gather: X_full    = all_gather(x_local)                   (stand-alone pull, used for wgrad re-gather)
//
// One persistent launch does both jobs:
//   * AG+GEMM (transfer overlapped with the math tile by tile): a few "copy warps" per CTA pull the peers' row chunks
//     over NVLink (16-byte P2P loads from the peers' symmetric buffers) into the local gathered buffer, publishing one
//     ready-flag per 128-row block; the wgmma GEMM main loop (gemm_sm90.cuh) runs in the same CTAs and its TMA producer
//     only waits for the flag of the A row-block it is about to load.  Tiles are ordered local chunk first, then chunks
//     in arrival order, so compute never idles while data is in flight.
//   * GEMM+RS (transfer NOT overlapped with the math): every CTA runs the wgmma GEMM, writing bf16 partial tiles into a
//     local symmetric buffer, chunk by chunk starting with the chunk owned by rank+1 (own chunk last); the last
//     warpgroup to finish a chunk signals its owner.  After the GEMM, each rank waits until every peer has finished its
//     chunk and reduces it straight out of the NVSwitch with multimem.ld_reduce (in-switch fp32 accumulation; P2P loads
//     + adds when no multicast mapping exists).
//   * cross-GPU ordering uses release/acquire at .sys scope on 32-bit epoch flags that live in symmetric memory; data
//     written through the generic proxy and later read by TMA is fenced with fence.proxy.async on both sides.
//
// These replace the reference's `dist.all_gather` + `F.linear` / `F.linear` + `dist.reduce_scatter` pairs
// (shardformer/layer/_operation.py:562-566, 737-751) and its python ring variants (`_ring_as_gather`,
// `_ring_as_reducescatter`): no NCCL call on these paths.
#include <stdio.h>
#include <stdlib.h>

#include "gemm_sm90.cuh"

using namespace sm90;

namespace {

constexpr int BLOCK_M = gemm90::BM;
constexpr int FIRST_COPY_WARP = gemm90::NUM_THREADS / 32;
// warps 0..8 = GEMM roles (gemm_sm90.cuh), warps 9..10 = NVLink pull (AG) / extra reduce lanes (RS)
constexpr int NUM_THREADS = gemm90::NUM_THREADS + 64;
constexpr int COPY_WARPS = 2;
constexpr int COPY_SEG = 8;           // a 128-row block is pulled as 8 segments of 16 rows by different warps
constexpr int GROUP_M = 8;
constexpr int MAX_RANKS = 16;

// flag slots (uint32) inside every rank's symmetric flag page
constexpr int SLOT_IN_READY = 0;                 // [MAX_RANKS]  peer p wrote: "my input buffer holds epoch e"
constexpr int SLOT_PULL_DONE = MAX_RANKS;        // [MAX_RANKS]  peer p wrote: "I finished reading your buffer (epoch e)"
constexpr int SLOT_CHUNK_DONE = 2 * MAX_RANKS;   // [MAX_RANKS]  peer p wrote: "my partial of YOUR chunk is complete"
constexpr int SLOT_LOCAL = 3 * MAX_RANKS;        // local scratch counters (never written by peers): [0..3]

struct CommParams {
  int rank, world;
  uint32_t epoch;
  int n_copy_ctas;                 // (unused by the fused kernels; CTAs of the stand-alone all-gather)
  int rows_per_chunk;              // T / world
  const void* peer_in[MAX_RANKS];  // AG: peers' symmetric input buffers [rows_per_chunk, ld_in]
  uint32_t* peer_flags[MAX_RANKS]; // every rank's flag page (index = rank)
  void* gathered;                  // AG: local [T, ld_in] gathered buffer (TMA source of A)
  int ld_in;                       // elements per row of the gathered / input buffers
  uint32_t* ready;                 // AG: local per-row-block ready flags [T / 128]
  uint32_t* block_counter;         // AG: local per-row-block segment arrival counters [T / 128]
  // RS
  const void* peer_part[MAX_RANKS];  // peers' symmetric partial buffers [T, ldc]
  const void* mc_part;               // multicast address of the partial buffer (or null)
  void* out;                         // RS: local output [rows_per_chunk, ld_out]
  int ld_out;
  uint32_t* chunk_counter;           // RS: local per-chunk arrival counters [world]
  int out_dtype;
};

struct GemmParams {
  int M, N, K;
  int ldc;
  int a_mn_major, b_mn_major;
  void* C;          // RS: local partial buffer (bf16); AG: output
  int out_dtype;
};

// ------------------------------------------------------------------------------------------- flag helpers
SM90_DEVICE void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
SM90_DEVICE uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SM90_DEVICE void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
SM90_DEVICE uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SM90_DEVICE void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
SM90_DEVICE bool epoch_reached(uint32_t v, uint32_t epoch) { return (int32_t)(v - epoch) >= 0; }

// Bounded spin on an epoch flag: a peer that never arrives (crashed rank, mismatched call sequence) must not hang the
// GPU forever - after ~20 s the kernel reports and traps, which surfaces as a CUDA error in the host process.
constexpr long long SPIN_TIMEOUT_CYCLES = 40LL * 1000 * 1000 * 1000;
template <bool SYS>
SM90_DEVICE void wait_epoch(const uint32_t* flag, uint32_t epoch) {
  if (epoch_reached(SYS ? ld_acquire_sys(flag) : ld_acquire_gpu(flag), epoch)) return;
  const long long t0 = clock64();
  uint32_t it = 0;
  while (!epoch_reached(SYS ? ld_acquire_sys(flag) : ld_acquire_gpu(flag), epoch)) {
    __nanosleep(100);
    if ((++it & 0x3fff) == 0 && clock64() - t0 > SPIN_TIMEOUT_CYCLES) {
      printf("[cb200 fused comm] timeout waiting for epoch %u on flag %p (have %u), block %d\n", epoch, (const void*)flag,
             *flag, (int)blockIdx.x);
      __trap();
    }
  }
}

SM90_DEVICE uint4 ld_peer_16B(const void* p) {
  uint4 r;
  asm volatile("ld.global.relaxed.sys.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
// in-switch reduction of 8 bf16 values held at the same offset on every rank (fp32 accumulate inside the NVSwitch)
SM90_DEVICE uint4 multimem_ld_reduce_bf16x8(const void* mc_addr) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc_addr) : "memory");
  return r;
}

SM90_DEVICE void tile_coords_rot(int tile, int m_blocks, int n_blocks, int m_rot, int& m_blk, int& n_blk) {
  const int tiles_per_group = GROUP_M * n_blocks;
  const int group = tile / tiles_per_group;
  const int first_m = group * GROUP_M;
  const int gsize = min(m_blocks - first_m, GROUP_M);
  const int in_group = tile - group * tiles_per_group;
  int m = first_m + in_group % gsize;
  n_blk = in_group / gsize;
  m_blk = (m + m_rot) % m_blocks;     // rotate so the preferred chunk's row blocks come first
}

SM90_DEVICE void ag_pull_warps(const CommParams& c, uint32_t* my_flags, int warp, int lane, int blocks_per_chunk) {
  // ================================================================ AG: NVLink pull by the copy warps of ALL CTAs
  if (blockIdx.x == 0 && warp == FIRST_COPY_WARP && lane < c.world)   // announce: my input buffer is valid for this epoch
    st_release_sys(c.peer_flags[lane] + SLOT_IN_READY + c.rank, c.epoch);
  const int vec_per_row = c.ld_in / 8;                  // 16-byte vectors per row
  const int copy_warp = (int)blockIdx.x * COPY_WARPS + (warp - FIRST_COPY_WARP);
  const int n_copy_warps = (int)gridDim.x * COPY_WARPS;
  const int units_per_chunk = blocks_per_chunk * COPY_SEG;
  const int seg_rows = BLOCK_M / COPY_SEG;
  const size_t seg_vec = (size_t)seg_rows * vec_per_row;
  int cur_src = -1;
  for (int u = copy_warp; u < units_per_chunk * c.world; u += n_copy_warps) {
    const int step = u / units_per_chunk;                // chunks in order rank, rank+1, ...
    const int src = (c.rank + step) % c.world;
    const int in_chunk = u - step * units_per_chunk;
    const int sb = in_chunk / COPY_SEG, seg = in_chunk - sb * COPY_SEG;
    if (src != cur_src) {
      if (src != c.rank) {
        if (lane == 0)
          wait_epoch<true>(my_flags + SLOT_IN_READY + src, c.epoch);
        __syncwarp();
      }
      cur_src = src;
    }
    const uint4* sp = reinterpret_cast<const uint4*>(c.peer_in[src]) + ((size_t)sb * BLOCK_M + seg * seg_rows) * vec_per_row;
    uint4* dp = reinterpret_cast<uint4*>(c.gathered) +
                ((size_t)src * c.rows_per_chunk + (size_t)sb * BLOCK_M + seg * seg_rows) * vec_per_row;
    size_t i = lane;
    for (; i + 15 * 32 < seg_vec; i += 16 * 32) {        // 16 independent 16-byte loads in flight per lane
      uint4 t[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) t[j] = ld_peer_16B(sp + i + j * 32);
#pragma unroll
      for (int j = 0; j < 16; ++j) dp[i + j * 32] = t[j];
    }
    for (; i + 7 * 32 < seg_vec; i += 8 * 32) {
      uint4 t[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t[j] = ld_peer_16B(sp + i + j * 32);
#pragma unroll
      for (int j = 0; j < 8; ++j) dp[i + j * 32] = t[j];
    }
    for (; i < seg_vec; i += 32) dp[i] = ld_peer_16B(sp + i);
    fence_proxy_async_global();          // generic-proxy writes -> visible to TMA (async proxy) readers
    __threadfence();
    __syncwarp();
    if (lane == 0) {
      const int blk = src * blocks_per_chunk + sb;
      const uint32_t got = atomicAdd(c.block_counter + blk, 1u) + 1;
      if (got == (uint32_t)COPY_SEG) {
        c.block_counter[blk] = 0;
        __threadfence();
        st_release_gpu(c.ready + blk, c.epoch);
      }
    }
  }
  // tell every peer that this rank no longer reads its input buffer (last copy warp to finish signals)
  if (lane == 0) {
    const uint32_t done = atomicAdd(my_flags + SLOT_LOCAL, 1u) + 1;
    if (done == (uint32_t)n_copy_warps) {
      my_flags[SLOT_LOCAL] = 0;
      __threadfence_system();
      for (int r = 0; r < c.world; ++r) st_release_sys(c.peer_flags[r] + SLOT_PULL_DONE + c.rank, c.epoch);
    }
  }
}

// Reduce-scatter tail (GEMM+RS): after every peer signalled its partial of MY chunk, sum the chunk out of all partial
// buffers (in-switch multimem reduction when a multicast mapping exists) and release the partial buffers.
SM90_DEVICE void rs_reduce_phase(const GemmParams& p, const CommParams& c, uint32_t* my_flags) {
  // ================================================================== RS: reduce MY chunk out of all partial buffers
  if (threadIdx.x < c.world) {
    wait_epoch<true>(my_flags + SLOT_CHUNK_DONE + threadIdx.x, c.epoch);
  }
  __syncthreads();
  const int vec_per_row = p.N / 8;
  const size_t row0 = (size_t)c.rank * c.rows_per_chunk;
  const size_t nvec = (size_t)c.rows_per_chunk * vec_per_row;
  const size_t ldc_vec = p.ldc / 8;
  const size_t stride = (size_t)gridDim.x * NUM_THREADS;
  for (size_t i0 = (size_t)blockIdx.x * NUM_THREADS + threadIdx.x; i0 < nvec; i0 += 4 * stride) {
    uint4 sum[4];
    size_t dst_off[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {                           // 4 independent switch reductions in flight per thread
      const size_t i = i0 + u * stride;
      if (i >= nvec) { dst_off[u] = (size_t)-1; continue; }
      const size_t r = i / vec_per_row, cv = i - r * vec_per_row;
      const size_t src_off = (row0 + r) * ldc_vec + cv;     // 16-byte units inside the partial buffer
      dst_off[u] = r * (c.ld_out / 8) + cv;
      if (c.mc_part) {
        sum[u] = multimem_ld_reduce_bf16x8(reinterpret_cast<const uint4*>(c.mc_part) + src_off);
      } else {
        float accf[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int rk = 0; rk < c.world; ++rk) {
          const int src = (c.rank + rk) % c.world;
          Vec16<__nv_bfloat16> v;
          v.raw = ld_peer_16B(reinterpret_cast<const uint4*>(c.peer_part[src]) + src_off);
#pragma unroll
          for (int k = 0; k < 8; ++k) accf[k] += v.get(k);
        }
        Vec16<__nv_bfloat16> o;
#pragma unroll
        for (int k = 0; k < 8; ++k) o.set(k, accf[k]);
        sum[u] = o.raw;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (dst_off[u] != (size_t)-1) reinterpret_cast<uint4*>(c.out)[dst_off[u]] = sum[u];
  }
  // everyone may now overwrite their partial buffer again: last CTA of this rank signals all peers
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t done = atomicAdd(my_flags + SLOT_LOCAL + 1, 1u) + 1;
    if (done == gridDim.x) {
      my_flags[SLOT_LOCAL + 1] = 0;
      __threadfence_system();
      for (int r = 0; r < c.world; ++r) st_release_sys(c.peer_flags[r] + SLOT_PULL_DONE + c.rank, c.epoch);
    }
  }
}

// MODE 0: all-gather + GEMM.  MODE 1: GEMM + reduce-scatter.
// The GEMM roles are those of gemm_sm90.cuh (warps 0..7 consumers, warp 8 producer); the tile order is rotated so the
// preferred chunk comes first.  AG: the producer waits for the ready flag of the A row-block it is about to load.
// RS: after storing its half of a partial tile a consumer warpgroup counts it for the chunk; the last one of a chunk
// tells the chunk's owner.
template <int MODE> struct FusedProb {
  GemmParams p;
  CommParams c;
  int m_blocks, n_blocks, m_rot, blocks_per_chunk;
  SM90_DEVICE int num_tiles() const { return m_blocks * n_blocks; }
  SM90_DEVICE gemm90::Tile tile(int idx) const {
    int m_blk, n_blk;
    tile_coords_rot(idx, m_blocks, n_blocks, m_rot, m_blk, n_blk);
    gemm90::Tile t;
    t.a_mn0 = m_blk * BLOCK_M; t.a_k0 = 0;
    t.b_mn0 = n_blk * gemm90::BN; t.b_k0 = 0;
    t.k_blocks = (p.K + 63) / 64;
    t.row0 = m_blk * BLOCK_M; t.row_lim = p.M;
    t.col0 = n_blk * gemm90::BN; t.col_lim = p.N;
    t.c_base = 0;
    return t;
  }
  SM90_DEVICE void before_load(int, const gemm90::Tile& t) const {
    if (MODE == 0) {
      wait_epoch<false>(c.ready + t.a_mn0 / BLOCK_M, c.epoch);    // the A rows of this tile landed in `gathered`
      fence_proxy_async_global();
    }
  }
  SM90_DEVICE void after_store(int, const gemm90::Tile& t, int wg) const {
    if (MODE != 1) return;
    // publish: this warpgroup's half of the partial tile is globally visible; count tiles per chunk
    __threadfence_system();
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    if ((threadIdx.x & 127) == 0) {
      const int chunk = (t.a_mn0 / BLOCK_M) / blocks_per_chunk;
      const uint32_t got = atomicAdd(c.chunk_counter + chunk, 1u) + 1;
      const uint32_t need = (uint32_t)blocks_per_chunk * n_blocks * 2;   // 2 consumer warpgroups per tile
      if (got == need) {
        c.chunk_counter[chunk] = 0;
        __threadfence_system();
        st_release_sys(c.peer_flags[chunk] + SLOT_CHUNK_DONE + c.rank, c.epoch);
      }
    }
  }
};

template <int MODE, int A_MN, int B_MN, int KIND>
__global__ void __launch_bounds__(NUM_THREADS, 1)
fused_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const GemmParams p, const CommParams c) {
  extern __shared__ uint8_t smem_raw[];
  const gemm90::Smem s = gemm90::carve(smem_raw);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  FusedProb<MODE> prob;
  prob.p = p;
  prob.c = c;
  prob.m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M;
  prob.n_blocks = (p.N + gemm90::BN - 1) / gemm90::BN;
  prob.blocks_per_chunk = c.rows_per_chunk / BLOCK_M;
  // AG: local chunk first.  RS: start with the chunk owned by rank+1, own chunk last.
  prob.m_rot = MODE == 0 ? c.rank * prob.blocks_per_chunk : ((c.rank + 1) % c.world) * prob.blocks_per_chunk;
  uint32_t* my_flags = c.peer_flags[c.rank];
  if (threadIdx.x == 0) gemm90::init_barriers(s);
  if (warp == gemm90::PRODUCER_WARP && lane == 0) {
    prefetch_tensormap(&tmap_a);
    prefetch_tensormap(&tmap_b);
  }
  __syncthreads();
  const int num_tiles = prob.num_tiles();
  if (warp >= FIRST_COPY_WARP) {
    if (MODE == 0) ag_pull_warps(c, my_flags, warp, lane, prob.blocks_per_chunk);
  } else if (warp == gemm90::PRODUCER_WARP) {
    gemm90::producer<KIND, A_MN, B_MN>(&tmap_a, &tmap_b, prob, s, num_tiles);
  } else {
    const gemm90::Epilogue e{p.C, p.ldc, p.out_dtype, 0, nullptr, nullptr};
    gemm90::consumer<KIND, A_MN, B_MN>(prob, s, e, num_tiles);
  }
  __syncthreads();
  if (MODE == 1) rs_reduce_phase(p, c, my_flags);
}

// Stand-alone all-gather by P2P pull (every CTA is a copy CTA).
__global__ void __launch_bounds__(256) all_gather_pull_kernel(const CommParams c) {
  uint32_t* my_flags = c.peer_flags[c.rank];
  if (blockIdx.x == 0 && threadIdx.x < c.world)
    st_release_sys(c.peer_flags[threadIdx.x] + SLOT_IN_READY + c.rank, c.epoch);
  const size_t vec_per_chunk = (size_t)c.rows_per_chunk * (c.ld_in / 8);
  for (int step = 0; step < c.world; ++step) {
    const int src = (c.rank + step) % c.world;
    if (step > 0) {
      if (threadIdx.x == 0)
        wait_epoch<true>(my_flags + SLOT_IN_READY + src, c.epoch);
      __syncthreads();
    }
    const uint4* s = reinterpret_cast<const uint4*>(c.peer_in[src]);
    uint4* d = reinterpret_cast<uint4*>(c.gathered) + (size_t)src * vec_per_chunk;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < vec_per_chunk; i += (size_t)gridDim.x * blockDim.x)
      d[i] = ld_peer_16B(s + i);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t done = atomicAdd(my_flags + SLOT_LOCAL + 2, 1u) + 1;
    if (done == gridDim.x) {
      my_flags[SLOT_LOCAL + 2] = 0;
      __threadfence_system();
      for (int r = 0; r < c.world; ++r) st_release_sys(c.peer_flags[r] + SLOT_PULL_DONE + c.rank, c.epoch);
    }
  }
}

// Stand-alone reduce-scatter over symmetric memory: every rank has written its full [world * rows_per_chunk, ld] input
// into its symmetric buffer; rank r sums chunk r over all ranks (fp32 accumulation: in-switch `multimem.ld_reduce` when a
// multicast mapping exists, otherwise 16-byte P2P loads) and writes it to `out`.  ELEM: 0 = bf16, 1 = fp32.
SM90_DEVICE uint4 multimem_ld_reduce_f32x4(const void* mc_addr) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc_addr) : "memory");
  return r;
}

template <int ELEM>
__global__ void __launch_bounds__(256) reduce_scatter_kernel(const CommParams c, size_t vec_per_chunk) {
  uint32_t* my_flags = c.peer_flags[c.rank];
  // publish "my input buffer is complete" and wait for every peer's
  if (blockIdx.x == 0 && threadIdx.x < c.world) st_release_sys(c.peer_flags[threadIdx.x] + SLOT_IN_READY + c.rank, c.epoch);
  if (threadIdx.x < c.world)
    wait_epoch<true>(my_flags + SLOT_IN_READY + threadIdx.x, c.epoch);
  __syncthreads();
  const size_t base = (size_t)c.rank * vec_per_chunk;          // 16-byte units
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < vec_per_chunk; i0 += 8 * stride) {
    uint4 sum[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const size_t i = i0 + u * stride;
      if (i >= vec_per_chunk) continue;
      if (c.mc_part) {
        const uint4* a = reinterpret_cast<const uint4*>(c.mc_part) + base + i;
        sum[u] = ELEM == 0 ? multimem_ld_reduce_bf16x8(a) : multimem_ld_reduce_f32x4(a);
      } else if (ELEM == 0) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int rk = 0; rk < c.world; ++rk) {
          Vec16<__nv_bfloat16> v;
          v.raw = ld_peer_16B(reinterpret_cast<const uint4*>(c.peer_part[(c.rank + rk) % c.world]) + base + i);
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] += v.get(k);
        }
        Vec16<__nv_bfloat16> o;
#pragma unroll
        for (int k = 0; k < 8; ++k) o.set(k, acc[k]);
        sum[u] = o.raw;
      } else {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int rk = 0; rk < c.world; ++rk) {
          const uint4 v = ld_peer_16B(reinterpret_cast<const uint4*>(c.peer_part[(c.rank + rk) % c.world]) + base + i);
          acc.x += __uint_as_float(v.x); acc.y += __uint_as_float(v.y);
          acc.z += __uint_as_float(v.z); acc.w += __uint_as_float(v.w);
        }
        sum[u] = make_uint4(__float_as_uint(acc.x), __float_as_uint(acc.y), __float_as_uint(acc.z), __float_as_uint(acc.w));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const size_t i = i0 + u * stride;
      if (i < vec_per_chunk) reinterpret_cast<uint4*>(c.out)[i] = sum[u];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t done = atomicAdd(my_flags + SLOT_LOCAL + 2, 1u) + 1;
    if (done == gridDim.x) {
      my_flags[SLOT_LOCAL + 2] = 0;
      __threadfence_system();
      for (int r = 0; r < c.world; ++r) st_release_sys(c.peer_flags[r] + SLOT_PULL_DONE + c.rank, c.epoch);
    }
  }
}

// Ulysses (DeepSpeed sequence-parallel) layout switch as ONE pull kernel over peer memory, q / k / v segments together:
//   mode 0 "gather sequence, scatter heads":  in  [B * Sl, ld_in]  (all heads of my sequence shard)
//                                             out [B * sp * Sl, ld_out] (my head slice of the whole sequence); for segment s
//                                             out[(b * sp + src) * Sl + t, out_base[s] + c] = in_src[b * Sl + t, in_base[s] + me * ncols[s] + c]
//   mode 1 "scatter sequence, gather heads":  in  [B * sp * Sl, ld_in], out [B * Sl, ld_out];
//                                             out[b * Sl + t, out_base[s] + src * ncols[s] + c] = in_src[(b * sp + me) * Sl + t, in_base[s] + c]
// Replaces the reference's three `all_to_all` calls before attention and the one after it
// (`shardformer/modeling/llama.py:522-526,595-600`, `layer/_operation.py:1082-1153`) plus their chunk / cat copies.
struct A2ASeg {
  int in_base, out_base, ncols;          // in 16-byte vectors
};
struct A2AParams {
  int mode, B, Sl, n_seg, ld_in, ld_out; // leading dimensions in 16-byte vectors
  A2ASeg seg[3];
  void* out;
};

__global__ void __launch_bounds__(256) ulysses_a2a_kernel(const CommParams c, const A2AParams a) {
  uint32_t* my_flags = c.peer_flags[c.rank];
  if (blockIdx.x == 0 && threadIdx.x < c.world)
    st_release_sys(c.peer_flags[threadIdx.x] + SLOT_IN_READY + c.rank, c.epoch);
  const int sp = c.world, me = c.rank;
  uint4* out = reinterpret_cast<uint4*>(a.out);
  for (int step = 0; step < sp; ++step) {
    const int src = (me + step) % sp;
    if (step > 0) {
      if (threadIdx.x == 0) wait_epoch<true>(my_flags + SLOT_IN_READY + src, c.epoch);
      __syncthreads();
    }
    const uint4* in = reinterpret_cast<const uint4*>(c.peer_in[src]);
    for (int s = 0; s < a.n_seg; ++s) {
      const A2ASeg sg = a.seg[s];
      const size_t per_b = (size_t)a.Sl * sg.ncols;
      const size_t total = (size_t)a.B * per_b;
      for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / per_b);
        const size_t r = i - (size_t)b * per_b;
        const int t = (int)(r / sg.ncols), cv = (int)(r - (size_t)t * sg.ncols);
        size_t in_off, out_off;
        if (a.mode == 0) {
          in_off = ((size_t)b * a.Sl + t) * a.ld_in + sg.in_base + (size_t)me * sg.ncols + cv;
          out_off = (((size_t)b * sp + src) * a.Sl + t) * a.ld_out + sg.out_base + cv;
        } else {
          in_off = (((size_t)b * sp + me) * a.Sl + t) * a.ld_in + sg.in_base + cv;
          out_off = ((size_t)b * a.Sl + t) * a.ld_out + sg.out_base + (size_t)src * sg.ncols + cv;
        }
        out[out_off] = ld_peer_16B(in + in_off);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t done = atomicAdd(my_flags + SLOT_LOCAL + 3, 1u) + 1;
    if (done == gridDim.x) {
      my_flags[SLOT_LOCAL + 3] = 0;
      __threadfence_system();
      for (int r = 0; r < c.world; ++r) st_release_sys(c.peer_flags[r] + SLOT_PULL_DONE + c.rank, c.epoch);
    }
  }
}

// Wait until every peer has finished reading this rank's symmetric buffers of `epoch` (buffer-reuse guard).
__global__ void wait_pull_done_kernel(uint32_t* my_flags, int world, uint32_t epoch) {
  if (threadIdx.x < world)
    wait_epoch<true>(my_flags + SLOT_PULL_DONE + threadIdx.x, epoch);
}

template <int MODE, int A_MN, int B_MN, int KIND>
int launch_fused_k(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, const CommParams& c,
                   cudaStream_t stream) {
  constexpr int SMEM = gemm90::SMEM_BYTES;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(fused_gemm_kernel<MODE, A_MN, B_MN, KIND>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  // persistent grid: ALL CTAs must be co-resident (flag spinning) -> exactly one CTA per SM
  fused_gemm_kernel<MODE, A_MN, B_MN, KIND><<<cb_num_sms(), NUM_THREADS, SMEM, stream>>>(ta, tb, p, c);
  return (int)cudaGetLastError();
}

template <int MODE>
int launch_fused(const void* A, const void* B, int M, int N, int K, int lda, int ldb, int a_mn, int b_mn, int in_dtype,
                 GemmParams p, const CommParams& c, cudaStream_t stream) {
  CUtensorMap ta, tb;
  const bool bf16 = in_dtype == CB_BF16;
  int r = gemm90::tmap16(&ta, A, a_mn, M, K, lda, bf16);
  if (r) return 1000 + r;
  r = gemm90::tmap16(&tb, B, b_mn, N, K, ldb, bf16);
  if (r) return 2000 + r;
#define CB_F(A_, B_)                                                                     \
  return bf16 ? launch_fused_k<MODE, A_, B_, gemm90::K_BF16>(ta, tb, p, c, stream)       \
              : launch_fused_k<MODE, A_, B_, gemm90::K_F16>(ta, tb, p, c, stream)
  if (!a_mn && !b_mn) CB_F(0, 0);
  if (!a_mn && b_mn) CB_F(0, 1);
  if (a_mn && !b_mn) CB_F(1, 0);
  CB_F(1, 1);
#undef CB_F
}

}  // namespace

extern "C" {

int cb_fused_max_ranks() { return MAX_RANKS; }
int cb_fused_flag_words() { return 5 * MAX_RANKS; }

// Y[T, N] = gather(x)[T, K] (x) B.   peer_in[r] = rank r's symmetric x_local buffer; `gathered` is a local [T, ld_in]
// buffer (returned to the caller for the backward pass); `ready` is a local uint32[T/128] array.
// b_mn_major == 0: B is [N, K] (fwd: W[N_local, K]);  == 1: B is stored [K, N] (dgrad: W[K=N_out_local, N=K_in]).
int cb_ag_gemm(const void* const* peer_in, uint32_t* const* peer_flags, void* gathered, uint32_t* ready,
               uint32_t* block_counter,
               const void* B, void* Y, int T, int N, int K, int ldb, int ldy, int b_mn_major, int in_dtype,
               int rank, int world, uint32_t epoch, int n_copy_ctas, int block_n, cudaStream_t stream) {
  if (world > MAX_RANKS || T % (world * BLOCK_M) != 0 || K % 8 != 0) return (int)cudaErrorInvalidValue;
  CommParams c{};
  c.rank = rank; c.world = world; c.epoch = epoch; c.n_copy_ctas = n_copy_ctas; c.rows_per_chunk = T / world;
  for (int r = 0; r < world; ++r) { c.peer_in[r] = peer_in[r]; c.peer_flags[r] = peer_flags[r]; }
  c.gathered = gathered; c.ld_in = K; c.ready = ready; c.block_counter = block_counter;
  GemmParams p{};
  p.M = T; p.N = N; p.K = K; p.ldc = ldy; p.a_mn_major = 0; p.b_mn_major = b_mn_major; p.C = Y; p.out_dtype = in_dtype;
  (void)block_n;
  return launch_fused<0>(gathered, B, T, N, K, K, ldb, 0, b_mn_major, in_dtype, p, c, stream);
}

// y_local[T/world, N] = reduce_scatter_rows( A[T, K] (x) B ).  `part` is this rank's symmetric [T, N] partial buffer,
// peer_part[r] the peers' mappings of theirs, mc_part its multicast mapping (may be null).
int cb_gemm_rs(const void* A, const void* B, void* part, const void* const* peer_part, const void* mc_part,
               uint32_t* const* peer_flags, uint32_t* chunk_counter, void* out, int T, int N, int K, int lda, int ldb,
               int ld_out, int a_mn_major, int b_mn_major, int in_dtype, int rank, int world, uint32_t epoch,
               int block_n, cudaStream_t stream) {
  if (world > MAX_RANKS || T % (world * BLOCK_M) != 0 || N % 8 != 0) return (int)cudaErrorInvalidValue;
  CommParams c{};
  c.rank = rank; c.world = world; c.epoch = epoch; c.rows_per_chunk = T / world;
  for (int r = 0; r < world; ++r) { c.peer_part[r] = peer_part[r]; c.peer_flags[r] = peer_flags[r]; }
  c.mc_part = mc_part; c.out = out; c.ld_out = ld_out; c.chunk_counter = chunk_counter; c.out_dtype = in_dtype;
  GemmParams p{};
  p.M = T; p.N = N; p.K = K; p.ldc = N; p.a_mn_major = a_mn_major; p.b_mn_major = b_mn_major; p.C = part;
  p.out_dtype = in_dtype;
  (void)block_n;
  return launch_fused<1>(A, B, T, N, K, lda, ldb, a_mn_major, b_mn_major, in_dtype, p, c, stream);
}

int cb_all_gather_pull(const void* const* peer_in, uint32_t* const* peer_flags, void* gathered, int rows_per_chunk,
                       int ld_elems, int rank, int world, uint32_t epoch, int n_ctas, cudaStream_t stream) {
  if (world > MAX_RANKS || ld_elems % 8 != 0) return (int)cudaErrorInvalidValue;
  CommParams c{};
  c.rank = rank; c.world = world; c.epoch = epoch; c.rows_per_chunk = rows_per_chunk; c.ld_in = ld_elems;
  for (int r = 0; r < world; ++r) { c.peer_in[r] = peer_in[r]; c.peer_flags[r] = peer_flags[r]; }
  c.gathered = gathered;
  all_gather_pull_kernel<<<n_ctas, 256, 0, stream>>>(c);
  return (int)cudaGetLastError();
}

// out[chunk_bytes] = sum over ranks of (rank's symmetric buffer)[my chunk].  elem: 0 = bf16, 1 = fp32.
int cb_reduce_scatter(const void* const* peer_part, const void* mc_part, uint32_t* const* peer_flags, void* out,
                      int64_t chunk_bytes, int elem, int rank, int world, uint32_t epoch, int n_ctas,
                      cudaStream_t stream) {
  if (world > MAX_RANKS || chunk_bytes % 16 != 0) return (int)cudaErrorInvalidValue;
  CommParams c{};
  c.rank = rank; c.world = world; c.epoch = epoch;
  for (int r = 0; r < world; ++r) { c.peer_part[r] = peer_part[r]; c.peer_flags[r] = peer_flags[r]; }
  c.mc_part = mc_part; c.out = out;
  const size_t vec = (size_t)chunk_bytes / 16;
  if (elem == 0) reduce_scatter_kernel<0><<<n_ctas, 256, 0, stream>>>(c, vec);
  else reduce_scatter_kernel<1><<<n_ctas, 256, 0, stream>>>(c, vec);
  return (int)cudaGetLastError();
}

// Ulysses layout switch (see ulysses_a2a_kernel).  Column quantities are in ELEMENTS of `elem_bytes` and must be multiples
// of 16 bytes; peer_in[r] = rank r's symmetric input buffer.
int cb_ulysses_a2a(const void* const* peer_in, uint32_t* const* peer_flags, void* out, int mode, int B, int Sl, int n_seg,
                   const int* in_base, const int* out_base, const int* ncols, int ld_in, int ld_out, int elem_bytes,
                   int rank, int world, uint32_t epoch, int n_ctas, cudaStream_t stream) {
  if (world > MAX_RANKS || n_seg < 1 || n_seg > 3 || (mode != 0 && mode != 1)) return (int)cudaErrorInvalidValue;
  const int per = 16 / elem_bytes;
  CommParams c{};
  c.rank = rank; c.world = world; c.epoch = epoch;
  for (int r = 0; r < world; ++r) { c.peer_in[r] = peer_in[r]; c.peer_flags[r] = peer_flags[r]; }
  A2AParams a{};
  a.mode = mode; a.B = B; a.Sl = Sl; a.n_seg = n_seg; a.out = out;
  if (ld_in % per || ld_out % per) return (int)cudaErrorInvalidValue;
  a.ld_in = ld_in / per; a.ld_out = ld_out / per;
  for (int s = 0; s < n_seg; ++s) {
    if (in_base[s] % per || out_base[s] % per || ncols[s] % per) return (int)cudaErrorInvalidValue;
    a.seg[s].in_base = in_base[s] / per; a.seg[s].out_base = out_base[s] / per; a.seg[s].ncols = ncols[s] / per;
  }
  ulysses_a2a_kernel<<<n_ctas, 256, 0, stream>>>(c, a);
  return (int)cudaGetLastError();
}
int cb_wait_pull_done(uint32_t* my_flags, int world, uint32_t epoch, cudaStream_t stream) {
  wait_pull_done_kernel<<<1, 32, 0, stream>>>(my_flags, world, epoch);
  return (int)cudaGetLastError();
}

}  // extern "C"
