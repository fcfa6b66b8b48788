// Mixture-of-experts kernels for sm_90a.
//
//  (1) capacity-based dispatch / combine (+ cumsum) used by the legacy top-1 / top-2 MoE layer.  Behavioural parity:
//      reference extensions/csrc/kernel/cuda/moe_kernel.cu (moe_dispatch_fwd/bwd, moe_combine_fwd/bwd, cumsum_sub_one).
//  (2) router: fused softmax + top-k (+ renormalisation)  (reference: python `F.softmax` + `torch.topk` in
//      shardformer/modeling/{mixtral,deepseek}.py).
//  (3) dropless expert-parallel dispatch / combine fused with the NVLink transfer.  The reference exchanges split sizes
//      with an all_to_all, SYNCs to the host for the split lists, runs an uneven NCCL all_to_all, re-sorts the received
//      rows by local expert and repeats everything on the way back (shardformer/modeling/mixtral.py:123-208,
//      moe/_operation.py:all_to_all_uneven).  Here every rank
//        * histograms its routing choices and P2P-stores the histogram into every peer's symmetric count matrix,
//        * derives from the full count matrix the exact row offset of each (source rank, expert) segment in the OWNER's
//          receive buffer (layout [local expert][source rank][rows] -> already grouped for the grouped GEMM),
//        * stores its token rows straight into the owners' receive buffers over NVLink (16-byte stores), then raises a
//          release flag on every peer,
//        * and on the way back PULLS its k expert outputs per token from the owners' output buffers with 16-byte P2P
//          loads, doing the weighted combine on the fly.
//      No host synchronisation, no NCCL call, no re-sort.  Flags are epoch-valued words in a symmetric flag page.
#include <stdio.h>

#include "common.cuh"

namespace {

constexpr int MAX_PEERS = 16;

// ------------------------------------------------------------------------------------------------ (1) legacy kernels
// mask [s, e] int32 (0/1), dest_idx [s, e] int32 position inside the expert's capacity buffer (valid where mask != 0)
template <typename T>
__global__ void moe_dispatch_fwd_kernel(const T* __restrict__ tokens, T* __restrict__ expert_in, const int* __restrict__ mask,
                                        const int* __restrict__ dest_idx, int s, int e, int c, int h) {
  const int row = blockIdx.x;
  for (int j = 0; j < e; ++j) {
    if (!mask[row * e + j]) continue;
    const int pos = dest_idx[row * e + j];
    if (pos < 0 || pos >= c) continue;
    const T* src = tokens + (int64_t)row * h;
    T* dst = expert_in + ((int64_t)j * c + pos) * h;
    for (int i = threadIdx.x; i < h; i += blockDim.x) dst[i] = src[i];
  }
}

template <typename T>
__global__ void moe_dispatch_bwd_kernel(T* __restrict__ d_tokens, const T* __restrict__ d_expert, const int* __restrict__ mask,
                                        const int* __restrict__ dest_idx, int s, int e, int c, int h) {
  const int row = blockIdx.x;
  for (int i = threadIdx.x; i < h; i += blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j < e; ++j) {
      if (!mask[row * e + j]) continue;
      const int pos = dest_idx[row * e + j];
      if (pos < 0 || pos >= c) continue;
      acc += to_f32<T>(d_expert[((int64_t)j * c + pos) * h + i]);
    }
    d_tokens[(int64_t)row * h + i] = from_f32<T>(acc);
  }
}

template <typename T>
__global__ void moe_combine_fwd_kernel(const T* __restrict__ expert_out, T* __restrict__ out, const float* __restrict__ logits,
                                       const int* __restrict__ mask, const int* __restrict__ dest_idx, int s, int e, int c,
                                       int h) {
  const int row = blockIdx.x;
  for (int i = threadIdx.x; i < h; i += blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j < e; ++j) {
      if (!mask[row * e + j]) continue;
      const int pos = dest_idx[row * e + j];
      if (pos < 0 || pos >= c) continue;
      acc += logits[row * e + j] * to_f32<T>(expert_out[((int64_t)j * c + pos) * h + i]);
    }
    out[(int64_t)row * h + i] = from_f32<T>(acc);
  }
}

// d_expert[j, pos] = logits[row, j] * dy[row];  d_logits[row, j] = <dy[row], expert_out[j, pos]>
template <typename T>
__global__ void moe_combine_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ expert_out, T* __restrict__ d_expert,
                                       float* __restrict__ d_logits, const float* __restrict__ logits,
                                       const int* __restrict__ mask, const int* __restrict__ dest_idx, int s, int e, int c,
                                       int h) {
  const int row = blockIdx.x;
  __shared__ float red[64];
  for (int j = 0; j < e; ++j) {
    float dot = 0.f;
    const bool on = mask[row * e + j] != 0;
    const int pos = on ? dest_idx[row * e + j] : -1;
    if (on && pos >= 0 && pos < c) {
      const float w = logits[row * e + j];
      const int64_t off = ((int64_t)j * c + pos) * h;
      for (int i = threadIdx.x; i < h; i += blockDim.x) {
        const float g = to_f32<T>(dy[(int64_t)row * h + i]);
        dot += g * to_f32<T>(expert_out[off + i]);
        d_expert[off + i] = from_f32<T>(w * g);
      }
    }
    float v[1] = {dot};
    block_sum<1>(v, red);
    if (threadIdx.x == 0) d_logits[row * e + j] = v[0];
  }
}

// exclusive running count along dim 0 of an int32 [s, e] 0/1 mask, minus nothing: out = cumsum(mask, 0) - 1
__global__ void cumsum_sub_one_kernel(const int* __restrict__ in, int* __restrict__ out, int s, int e) {
  // one block per expert column; 1024 threads scan in chunks
  const int col = blockIdx.x;
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int base = 0; base < s; base += blockDim.x) {
    const int r = base + threadIdx.x;
    int v = r < s ? in[r * e + col] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    int pre = 0;
    for (int w = 0; w < warp; ++w) pre += warp_tot[w];
    const int incl = carry + pre + x;
    if (r < s) out[r * e + col] = incl - 1;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) {
      int tot = 0;
      for (int w = 0; w < nw; ++w) tot += warp_tot[w];
      carry += tot;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ (2) router
// logits [T, E] (any float type) -> topk weights fp32 [T, K], indices int32 [T, K]; one warp per token, E <= 256
template <typename T>
__global__ void router_topk_kernel(const T* __restrict__ logits, float* __restrict__ w_out, int* __restrict__ idx_out,
                                   float* __restrict__ probs_out, int tokens, int E, int K, int renorm, int pre_softmax) {
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= tokens) return;
  constexpr int PER = 8;  // 32 * 8 = 256 experts max
  float v[PER];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int e = lane + i * 32;
    v[i] = e < E ? to_f32<T>(logits[(int64_t)t * E + e]) : -INFINITY;
    mx = fmaxf(mx, v[i]);
  }
  mx = warp_max(mx);
  float p[PER];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    p[i] = (lane + i * 32) < E ? __expf(v[i] - mx) : 0.f;
    sum += p[i];
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    p[i] *= inv;
    if (probs_out && (lane + i * 32) < E) probs_out[(int64_t)t * E + lane + i * 32] = p[i];
  }
  // iterative arg-max top-k (ties -> lowest index, as torch.topk does for distinct values)
  float sel_sum = 0.f;
  float my_w = 0.f;
  int my_i = 0;
  for (int k = 0; k < K; ++k) {
    float best = -1.f;
    int bi = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = lane + i * 32;
      if (e < E && (p[i] > best || (p[i] == best && e < bi))) { best = p[i]; bi = e; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    sel_sum += best;
    if (lane == k) { my_w = best; my_i = bi; }
    if ((bi & 31) == lane) p[bi >> 5] = -2.f;  // remove from further rounds
  }
  if (lane < K) {
    w_out[(int64_t)t * K + lane] = renorm ? my_w / fmaxf(sel_sum, 1e-20f) : my_w;
    idx_out[(int64_t)t * K + lane] = my_i;
  }
}

// ------------------------------------------------------------------------------------------------ (3) fused EP
struct EpParams {
  void* rows[MAX_PEERS];        // symmetric row buffers (push target), capacity rows x H
  uint32_t* flags[MAX_PEERS];   // symmetric flag pages
  int* counts[MAX_PEERS];       // symmetric count matrices [world][E]
  int rank, world, E, n_local, capacity;
  int align;                    // every (owner, expert) segment starts on a multiple of this many rows (1 = packed)
  uint32_t epoch;
};

constexpr int SLOT_CNT = 0;                  // + src rank
constexpr int SLOT_ROWS = MAX_PEERS;         // + src rank
constexpr int SLOT_Y = 2 * MAX_PEERS;        // + src rank
constexpr int FLAG_WORDS = 4 * MAX_PEERS;

CB_DEVICE void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
CB_DEVICE uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
CB_DEVICE void spin_until(const uint32_t* p, uint32_t epoch) {
  // epochs only grow; a later epoch also satisfies the wait (the producer has moved on, data of this epoch landed)
  if ((int32_t)(ld_acquire_sys(p) - epoch) >= 0) return;
  const long long t0 = clock64();
  uint32_t it = 0;
  while ((int32_t)(ld_acquire_sys(p) - epoch) < 0) {
    __nanosleep(100);
    if ((++it & 0x3fff) == 0 && clock64() - t0 > 40LL * 1000 * 1000 * 1000) {   // ~20 s: a peer never arrived
      printf("[cb200 moe] timeout waiting for epoch %u on flag %p\n", epoch, (const void*)p);
      __trap();
    }
  }
}

// histogram of the routing choices: counts[e] += 1 for every (t, k)
__global__ void ep_histogram_kernel(const int* __restrict__ topk_idx, int n, int E, int* __restrict__ counts) {
  extern __shared__ int sh[];
  for (int i = threadIdx.x; i < E; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int e = topk_idx[i];
    if (e >= 0 && e < E) atomicAdd(&sh[e], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < E; i += blockDim.x)
    if (sh[i]) atomicAdd(&counts[i], sh[i]);
}

// one block: publish my histogram row to every peer, wait for all rows, derive offsets.
//   send_off[e]      : first row (in the owner's buffer) of MY segment for global expert e
//   local_counts[el] : rows of local expert el's segment, rounded up to p.align (int64, feeds the grouped GEMM offsets)
//   local_offs[el]   : inclusive cumsum (int32) of local_counts
//   real_counts[el]  : rows actually received for local expert el (the rest of the segment is padding)
//   meta[0] = total rows of the local layout (padding included), meta[1] = overflow flag
__global__ void ep_exchange_counts_kernel(EpParams p, const int* __restrict__ my_counts, int* __restrict__ send_off,
                                          int64_t* __restrict__ local_counts, int* __restrict__ local_offs,
                                          int* __restrict__ real_counts, int* __restrict__ meta) {
  const int E = p.E, W = p.world, R = p.rank;
  for (int peer = 0; peer < W; ++peer) {
    int* dst = p.counts[peer] + (int64_t)R * E;
    for (int e = threadIdx.x; e < E; e += blockDim.x) dst[e] = my_counts[e];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < W) st_release_sys(p.flags[threadIdx.x] + SLOT_CNT + R, p.epoch);
  if (threadIdx.x < W) spin_until(p.flags[R] + SLOT_CNT + threadIdx.x, p.epoch);
  __syncthreads();
  const int* all = p.counts[R];  // [W][E] now complete
  // per-expert totals and my prefix over source ranks
  extern __shared__ int sh[];   // tot[E], pre[E]
  int* tot = sh;
  int* pre = sh + E;
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    int t = 0, pr = 0;
    for (int r = 0; r < W; ++r) {
      const int c = all[r * E + e];
      if (r < R) pr += c;
      t += c;
    }
    tot[e] = t;
    pre[e] = pr;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const int owner_first = (e / p.n_local) * p.n_local;
    int base = 0;
    for (int e2 = owner_first; e2 < e; ++e2) base += (tot[e2] + p.align - 1) / p.align * p.align;
    send_off[e] = base + pre[e];
  }
  if (threadIdx.x == 0) {
    int run = 0;
    for (int el = 0; el < p.n_local; ++el) {
      const int c = tot[R * p.n_local + el];
      const int pc = (c + p.align - 1) / p.align * p.align;
      real_counts[el] = c;
      local_counts[el] = pc;
      run += pc;
      local_offs[el] = run;
    }
    meta[0] = run;
    meta[1] = run > p.capacity ? 1 : 0;
  }
  // overflow on ANY owner must stop every sender that targets it: check all owners
  for (int o = threadIdx.x; o < W; o += blockDim.x) {
    int run = 0;
    for (int el = 0; el < p.n_local; ++el) run += (tot[o * p.n_local + el] + p.align - 1) / p.align * p.align;
    if (run > p.capacity) atomicExch(&meta[1], 1);
  }
}

// one warp per (token, k) row: claim a slot in my segment of the owner's buffer and store the row there.
//   assign != 0 : slot = atomicAdd(cursor[e]) and pos[t,k] is written;  assign == 0 : pos[t,k] is reused (backward)
//   scale (optional) [T*K] : row is multiplied by scale[i] (combine backward: w * dout)
template <typename T>
__global__ void __launch_bounds__(256) ep_push_rows_kernel(EpParams p, const T* __restrict__ x, const int* __restrict__ topk_idx,
                                                           const float* __restrict__ scale, const int* __restrict__ send_off,
                                                           int* __restrict__ cursor, int* __restrict__ pos, int n_rows,
                                                           int K, int H, int64_t x_stride, int assign,
                                                           const int* __restrict__ meta, unsigned int* __restrict__ done_ctr) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const bool overflow = meta[1] != 0;
  constexpr int V = Vec16<T>::N;
  for (int i = blockIdx.x * warps_per_block + (threadIdx.x >> 5); i < n_rows && !overflow; i += gridDim.x * warps_per_block) {
    const int e = topk_idx[i];
    int dst_row;
    if (assign) {
      int slot = 0;
      if (lane == 0) slot = atomicAdd(&cursor[e], 1);
      slot = __shfl_sync(0xffffffffu, slot, 0);
      dst_row = send_off[e] + slot;
      if (lane == 0) pos[i] = dst_row;
    } else {
      dst_row = pos[i];
    }
    const int owner = e / p.n_local;
    const T* src = x + (int64_t)(i / K) * x_stride;
    T* dst = reinterpret_cast<T*>(p.rows[owner]) + (int64_t)dst_row * H;
    const float sc = scale ? scale[i] : 1.f;
    for (int c = lane * V; c < H; c += 32 * V) {
      Vec16<T> v;
      v.load(src + c);
      if (scale) {
#pragma unroll
        for (int j = 0; j < V; ++j) v.set(j, v.get(j) * sc);
      }
      v.store(dst + c);
    }
  }
  // completion: every thread fences its remote stores, last block raises the flags on every peer
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = (atomicAdd(done_ctr, 1u) == gridDim.x - 1);
  __syncthreads();
  if (last) {
    if (threadIdx.x == 0) *done_ctr = 0;
    __threadfence_system();
    if (threadIdx.x < p.world) st_release_sys(p.flags[threadIdx.x] + SLOT_ROWS + p.rank, p.epoch);
  }
}

// wait until every peer's flag in [slot, slot+world) reached `epoch`  (1 block)
__global__ void ep_wait_kernel(EpParams p, int slot) {
  if (threadIdx.x < p.world) spin_until(p.flags[p.rank] + slot + threadIdx.x, p.epoch);
}

// raise flag `slot + rank` on every peer (1 block) — stream-ordered after the producer kernels of this rank
__global__ void ep_signal_kernel(EpParams p, int slot) {
  __threadfence_system();
  if (threadIdx.x < p.world) st_release_sys(p.flags[threadIdx.x] + slot + p.rank, p.epoch);
}

// out[t] = sum_k w[t,k] * Y_owner[pos[t,k]]  (w == nullptr -> plain sum); optionally keeps the gathered rows.
// one warp per token; waits for the owners' "y ready" flags first.
template <typename T>
__global__ void __launch_bounds__(256) ep_pull_combine_kernel(EpParams p, const int* __restrict__ topk_idx,
                                                              const float* __restrict__ w, const int* __restrict__ pos,
                                                              T* __restrict__ out, T* __restrict__ ys_keep, int tokens,
                                                              int K, int H) {
  if (threadIdx.x < p.world) spin_until(p.flags[p.rank] + SLOT_Y + threadIdx.x, p.epoch);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  constexpr int V = Vec16<T>::N;
  for (int t = blockIdx.x * warps_per_block + (threadIdx.x >> 5); t < tokens; t += gridDim.x * warps_per_block) {
    for (int c = lane * V; c < H; c += 32 * V) {
      float acc[V];
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = 0.f;
      for (int k = 0; k < K; ++k) {
        const int i = t * K + k;
        const int e = topk_idx[i];
        const int owner = e / p.n_local;
        const T* src = reinterpret_cast<const T*>(p.rows[owner]) + (int64_t)pos[i] * H + c;
        Vec16<T> v;
        v.load_nc(src);
        if (ys_keep) v.store(ys_keep + (int64_t)i * H + c);
        const float wk = w ? w[i] : 1.f;
#pragma unroll
        for (int j = 0; j < V; ++j) acc[j] += wk * v.get(j);
      }
      Vec16<T> o;
#pragma unroll
      for (int j = 0; j < V; ++j) o.set(j, acc[j]);
      o.store(out + (int64_t)t * H + c);
    }
  }
}

inline EpParams make_ep(const void* const* rows, const void* const* flags, const void* const* counts, int rank, int world,
                        int E, int capacity, uint32_t epoch) {
  EpParams p;
  for (int i = 0; i < MAX_PEERS; ++i) {
    p.rows[i] = i < world && rows ? const_cast<void*>(rows[i]) : nullptr;
    p.flags[i] = i < world ? (uint32_t*)flags[i] : nullptr;
    p.counts[i] = i < world && counts ? (int*)counts[i] : nullptr;
  }
  p.rank = rank; p.world = world; p.E = E; p.n_local = E / world; p.capacity = capacity; p.epoch = epoch;
  p.align = 1;
  return p;
}

}  // namespace

// Copy the live part of a receive buffer into an autograd-owned tensor: rows of the padded local layout that hold a
// received row are copied, padding rows are zero-filled, nothing beyond the layout (the over-allocated rest of the
// buffer) is touched.  One warp per row, 16-byte chunks.
__global__ void __launch_bounds__(256) ep_take_rows_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src,
                                                            int row_vecs, const int* __restrict__ local_offs,
                                                            const int* __restrict__ real_counts, int n_local,
                                                            int max_rows) {
  const int total = min(local_offs[n_local - 1], max_rows);   // (an overflowing dispatch is reported by meta[1])
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < total; r += warps) {
    int lo = 0, hi = n_local - 1;            // first segment whose end is beyond r
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (local_offs[mid] > r) hi = mid; else lo = mid + 1;
    }
    const int start = lo ? local_offs[lo - 1] : 0;
    const bool live = r - start < real_counts[lo];
    uint4* d = dst + (int64_t)r * row_vecs;
    const uint4* s = src + (int64_t)r * row_vecs;
    if (live) {
      for (int i = lane; i < row_vecs; i += 32) d[i] = s[i];
    } else {
      for (int i = lane; i < row_vecs; i += 32) d[i] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

extern "C" {

int cb_moe_flag_words() { return FLAG_WORDS; }

// ---- legacy
int cb_moe_dispatch_fwd(const void* tokens, void* expert_in, const int* mask, const int* dest_idx, int s, int e, int c,
                        int h, int dtype, cudaStream_t st) {
  if (s == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    moe_dispatch_fwd_kernel<T><<<s, 256, 0, st>>>((const T*)tokens, (T*)expert_in, mask, dest_idx, s, e, c, h);
  });
  return CB_LAUNCH_CHECK();
}
int cb_moe_dispatch_bwd(void* d_tokens, const void* d_expert, const int* mask, const int* dest_idx, int s, int e, int c,
                        int h, int dtype, cudaStream_t st) {
  if (s == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    moe_dispatch_bwd_kernel<T><<<s, 256, 0, st>>>((T*)d_tokens, (const T*)d_expert, mask, dest_idx, s, e, c, h);
  });
  return CB_LAUNCH_CHECK();
}
int cb_moe_combine_fwd(const void* expert_out, void* out, const float* logits, const int* mask, const int* dest_idx,
                       int s, int e, int c, int h, int dtype, cudaStream_t st) {
  if (s == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    moe_combine_fwd_kernel<T><<<s, 256, 0, st>>>((const T*)expert_out, (T*)out, logits, mask, dest_idx, s, e, c, h);
  });
  return CB_LAUNCH_CHECK();
}
int cb_moe_combine_bwd(const void* dy, const void* expert_out, void* d_expert, float* d_logits, const float* logits,
                       const int* mask, const int* dest_idx, int s, int e, int c, int h, int dtype, cudaStream_t st) {
  if (s == 0) return 0;
  CB_DISPATCH_FLOAT(dtype, T, {
    moe_combine_bwd_kernel<T><<<s, 256, 0, st>>>((const T*)dy, (const T*)expert_out, (T*)d_expert, d_logits, logits,
                                                  mask, dest_idx, s, e, c, h);
  });
  return CB_LAUNCH_CHECK();
}
int cb_moe_cumsum_sub_one(const int* in, int* out, int s, int e, cudaStream_t st) {
  if (s == 0 || e == 0) return 0;
  cumsum_sub_one_kernel<<<e, 1024, 0, st>>>(in, out, s, e);
  return CB_LAUNCH_CHECK();
}

// ---- router
int cb_moe_router_topk(const void* logits, float* w_out, int* idx_out, float* probs_out, int tokens, int E, int K,
                       int renorm, int dtype, cudaStream_t st) {
  if (tokens == 0) return 0;
  if (E > 256 || K > 32 || K > E) return (int)cudaErrorInvalidValue;
  const int wpb = 8;
  CB_DISPATCH_FLOAT(dtype, T, {
    router_topk_kernel<T><<<(tokens + wpb - 1) / wpb, wpb * 32, 0, st>>>((const T*)logits, w_out, idx_out, probs_out,
                                                                         tokens, E, K, renorm, 0);
  });
  return CB_LAUNCH_CHECK();
}

// ---- fused EP
// counts_local / cursor: int[E] scratch (zeroed here); send_off int[E]; local_counts int64[n_local]; local_offs int[n_local];
// meta int[2]; pos int[T*K] (output)
int cb_moe_ep_dispatch(const void* x, const int* topk_idx, const void* const* rows, const void* const* flags,
                       const void* const* counts, int* counts_local, int* cursor, int* send_off, int64_t* local_counts,
                       int* local_offs, int* real_counts, int* meta, int* pos, unsigned int* done_ctr, int tokens, int K,
                       int H, int64_t x_stride, int E, int capacity, int align, int rank, int world, uint32_t epoch,
                       int dtype, cudaStream_t st) {
  if (world > MAX_PEERS || E % world != 0 || H % 8 != 0 || align < 1) return (int)cudaErrorInvalidValue;
  EpParams p = make_ep(rows, flags, counts, rank, world, E, capacity, epoch);
  p.align = align;
  const int n = tokens * K;
  cudaMemsetAsync(counts_local, 0, sizeof(int) * E, st);
  cudaMemsetAsync(cursor, 0, sizeof(int) * E, st);
  if (n > 0) {
    int g = (n + 1023) / 1024;
    if (g > cb_num_sms()) g = cb_num_sms();
    ep_histogram_kernel<<<g, 256, E * sizeof(int), st>>>(topk_idx, n, E, counts_local);
  }
  ep_exchange_counts_kernel<<<1, 256, 2 * E * sizeof(int), st>>>(p, counts_local, send_off, local_counts, local_offs,
                                                                 real_counts, meta);
  int grid = (n + 7) / 8;
  if (grid > cb_num_sms() * 4) grid = cb_num_sms() * 4;
  if (grid < 1) grid = 1;
  CB_DISPATCH_HALF(dtype, T, {
    ep_push_rows_kernel<T><<<grid, 256, 0, st>>>(p, (const T*)x, topk_idx, nullptr, send_off, cursor, pos, n, K, H,
                                                 x_stride, 1, meta, done_ctr);
  });
  ep_wait_kernel<<<1, 32, 0, st>>>(p, SLOT_ROWS);
  return CB_LAUNCH_CHECK();
}

// dst[r] = live row ? src[r] : 0 over the rows of the padded local layout (see ep_take_rows_kernel); row_bytes % 16 == 0
int cb_moe_ep_take_rows(void* dst, const void* src, int64_t row_bytes, const int* local_offs, const int* real_counts,
                        int n_local, int max_rows, cudaStream_t st) {
  if (row_bytes % 16 != 0 || n_local < 1) return (int)cudaErrorInvalidValue;
  ep_take_rows_kernel<<<cb_num_sms() * 4, 256, 0, st>>>((uint4*)dst, (const uint4*)src, (int)(row_bytes / 16), local_offs,
                                               real_counts, n_local, max_rows);
  return CB_LAUNCH_CHECK();
}

// push rows to already-known positions (combine backward: rows = scale[t,k] * x[t]) and wait for every peer's rows
int cb_moe_ep_push_known(const void* x, const int* topk_idx, const float* scale, const int* pos, const void* const* rows,
                         const void* const* flags, const int* meta, unsigned int* done_ctr, int tokens, int K, int H,
                         int64_t x_stride, int E, int rank, int world, uint32_t epoch, int dtype, cudaStream_t st) {
  if (world > MAX_PEERS || E % world != 0 || H % 8 != 0) return (int)cudaErrorInvalidValue;
  EpParams p = make_ep(rows, flags, nullptr, rank, world, E, 0, epoch);
  const int n = tokens * K;
  int grid = (n + 7) / 8;
  if (grid > cb_num_sms() * 4) grid = cb_num_sms() * 4;
  if (grid < 1) grid = 1;
  CB_DISPATCH_HALF(dtype, T, {
    ep_push_rows_kernel<T><<<grid, 256, 0, st>>>(p, (const T*)x, topk_idx, scale, nullptr, nullptr,
                                                 const_cast<int*>(pos), n, K, H, x_stride, 0, meta, done_ctr);
  });
  ep_wait_kernel<<<1, 32, 0, st>>>(p, SLOT_ROWS);
  return CB_LAUNCH_CHECK();
}

// signal "my output buffer is complete" then pull + combine.  rows[] here are the symmetric OUTPUT buffers.
int cb_moe_ep_combine(const int* topk_idx, const float* w, const int* pos, const void* const* rows,
                      const void* const* flags, void* out, void* ys_keep, int tokens, int K, int H, int E, int rank,
                      int world, uint32_t epoch, int dtype, cudaStream_t st) {
  if (world > MAX_PEERS || E % world != 0 || H % 8 != 0) return (int)cudaErrorInvalidValue;
  EpParams p = make_ep(rows, flags, nullptr, rank, world, E, 0, epoch);
  ep_signal_kernel<<<1, 32, 0, st>>>(p, SLOT_Y);
  int grid = (tokens + 7) / 8;
  if (grid > cb_num_sms() * 4) grid = cb_num_sms() * 4;
  if (grid < 1) grid = 1;
  CB_DISPATCH_HALF(dtype, T, {
    ep_pull_combine_kernel<T><<<grid, 256, 0, st>>>(p, topk_idx, w, pos, (T*)out, (T*)ys_keep, tokens, K, H);
  });
  return CB_LAUNCH_CHECK();
}

}  // extern "C"
