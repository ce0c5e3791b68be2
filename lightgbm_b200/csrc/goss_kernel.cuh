// goss_kernel.cuh — gradient-based one-side sampling on the device (sm_90a).
//
// Replaces: GOSSStrategy::Bagging / Helper (reference src/boosting/goss.hpp:30-77, :118-167): keep the rows whose
// |gradient * hessian| is among the top `top_rate` fraction, keep every other row with probability
// other_k / (n - top_k) and multiply the (gradient, hessian) of those by (n - top_k) / other_k; the kept rows, in
// ascending order, become the tree learner's bagging set (SetBaggingData).  The reference does this on the host, one
// chunk of rows per OpenMP thread with a per-chunk threshold and a sequential per-chunk RNG, and its own multi-GPU
// mode rejects it outright (src/boosting/cuda/nccl_gbdt.cpp:112-114).  Here: one exact global threshold by a 4-pass
// radix select over the float bit patterns, a counter-based uniform per row (a fixed function of (seed, iteration, row),
// independent of the launch geometry), and a stable compaction — so the bag never leaves HBM and its size is read by
// the prepare kernels from device memory (the captured per-tree graph is replayed unchanged).
// Parity with the reference is therefore statistical in WHICH small-gradient rows are drawn, exact in everything else:
// every row with |g*h| >= the k-th largest is kept, kept small-gradient rows are scaled by the same factor, the index
// list is ascending (tests/test_gpu_goss.py).
#pragma once
#include "partition_kernel.cuh"
#include "types.cuh"

namespace b200 {

struct GossState {
  uint32_t prefix, mask;        // radix select: bits of the threshold key decided so far
  uint32_t k_rem;               // rank still to resolve inside the current prefix bucket
  uint32_t threshold_key;       // float bits of the k-th largest |g*h|
  float multiply;               // (n - top_k) / other_k
  float prob;                   // other_k / (n - top_k)
  int32_t top_k, other_k;
};

struct GossArgs {
  float* grad; float* hess; int32_t n;
  uint32_t* hist;               // [256] bucket counts of the current pass
  GossState* st;
  uint32_t* flag_words;         // [ceil(n / 32)] keep bits
  int32_t* block_cnt;           // [gridDim.x]
  int32_t* bag;                 // [n] out: ascending kept row ids
  int32_t* bag_count;           // out: number of kept rows (device)
  double top_rate, other_rate;
  uint32_t seed, iter;
};

constexpr int kGossThreads = 256;

__device__ __forceinline__ uint32_t goss_key(float g, float h) { return __float_as_uint(fabsf(g * h)); }   // >= 0: uint order == float order

__global__ void __launch_bounds__(32) k_goss_begin(const GossArgs a) {
  if (threadIdx.x == 0) {
    GossState* s = a.st;
    // goss.hpp:130-136
    int top_k = static_cast<int>(a.n * a.top_rate); if (top_k < 1) top_k = 1;
    int other_k = static_cast<int>(a.n * a.other_rate);
    s->top_k = top_k; s->other_k = other_k;
    s->multiply = other_k > 0 ? static_cast<float>(a.n - top_k) / other_k : 0.f;
    s->prob = (a.n - top_k) > 0 ? static_cast<float>(static_cast<double>(other_k) / (a.n - top_k)) : 0.f;
    s->prefix = 0u; s->mask = 0u; s->k_rem = static_cast<uint32_t>(top_k);
  }
  for (int i = threadIdx.x; i < 256; i += 32) a.hist[i] = 0u;
}

// one radix pass (8 bits, most significant first): histogram of the next digit over the keys matching the prefix
__global__ void __launch_bounds__(kGossThreads) k_goss_hist(const GossArgs a, int shift) {
  __shared__ uint32_t s_h[256];
  s_h[threadIdx.x] = 0u;
  __syncthreads();
  const uint32_t prefix = a.st->prefix, mask = a.st->mask;
  for (int i = blockIdx.x * kGossThreads + threadIdx.x; i < a.n; i += gridDim.x * kGossThreads) {
    const uint32_t key = goss_key(a.grad[i], a.hess[i]);
    if ((key & mask) == prefix) atomicAdd(&s_h[(key >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (s_h[threadIdx.x]) atomicAdd(&a.hist[threadIdx.x], s_h[threadIdx.x]);
}

// walk the buckets from the top: the bucket in which the k-th largest key lies becomes the next digit of the threshold
__global__ void __launch_bounds__(32) k_goss_pick(const GossArgs a, int shift) {
  if (threadIdx.x == 0) {
    GossState* s = a.st;
    uint32_t k = s->k_rem, above = 0u; int b = 255;
    for (; b > 0; --b) {
      const uint32_t c = a.hist[b];
      if (above + c >= k) break;
      above += c;
    }
    s->prefix |= static_cast<uint32_t>(b) << shift;
    s->mask |= 255u << shift;
    s->k_rem = k - above;
    if (shift == 0) s->threshold_key = s->prefix;
  }
  __syncwarp();
  for (int i = threadIdx.x; i < 256; i += 32) a.hist[i] = 0u;
}

// keep flags (bit-packed, one ballot word per 32 rows), scaling of the sampled small-gradient rows, per-block counts
__global__ void __launch_bounds__(kGossThreads) k_goss_mark(const GossArgs a) {
  const GossState s = *a.st;
  int lo, hi;
  part_block_range(a.n, gridDim.x, blockIdx.x, &lo, &hi);
  const int lane = threadIdx.x & 31;
  int cnt = 0;
  for (int base = lo; base < hi; base += kGossThreads) {
    const int i = base + threadIdx.x;
    bool keep = false;
    if (i < hi) {
      const float g = a.grad[i], h = a.hess[i];
      if (goss_key(g, h) >= s.threshold_key) keep = true;
      else if (quant_uniform(a.seed, a.iter, static_cast<unsigned>(i), kGossStream) < static_cast<double>(s.prob)) {
        keep = true;
        a.grad[i] = g * s.multiply; a.hess[i] = h * s.multiply;          // goss.hpp:157-158
      }
    }
    const unsigned word = __ballot_sync(0xffffffffu, keep);
    if (lane == 0 && (i - lane) < hi) { a.flag_words[(i - lane) >> 5] = word; cnt += __popc(word); }
  }
  __shared__ int s_cnt[kGossThreads / 32];
  if (lane == 0) s_cnt[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kGossThreads / 32; ++w) t += s_cnt[w];
    a.block_cnt[blockIdx.x] = t;
  }
}

// stable compaction: ascending row ids of the kept rows; block 0 publishes the total
__global__ void __launch_bounds__(kGossThreads) k_goss_scatter(const GossArgs a) {
  __shared__ int s_before, s_total;
  __shared__ int s_red[kGossThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    int b = 0, t = 0;
    for (int j = 0; j < static_cast<int>(gridDim.x); ++j) { const int v = a.block_cnt[j]; if (j < static_cast<int>(blockIdx.x)) b += v; t += v; }
    s_before = b; s_total = t;
  }
  __syncthreads();
  if (blockIdx.x == 0 && tid == 0) *a.bag_count = s_total;
  int run = s_before;
  int lo, hi;
  part_block_range(a.n, gridDim.x, blockIdx.x, &lo, &hi);
  for (int base = lo; base < hi; base += kGossThreads) {
    const int i = base + tid;
    const int w0 = i - lane;
    const unsigned word = (w0 < hi) ? a.flag_words[w0 >> 5] : 0u;
    if (lane == 0) s_red[warp] = __popc(word);
    __syncthreads();
    int wbefore = 0, tile = 0;
#pragma unroll
    for (int w = 0; w < kGossThreads / 32; ++w) { const int v = s_red[w]; if (w < warp) wbefore += v; tile += v; }
    if (i < hi && ((word >> lane) & 1u)) a.bag[run + wbefore + __popc(word & ((1u << lane) - 1u))] = i;
    run += tile;
    __syncthreads();
  }
}

}  // namespace b200
