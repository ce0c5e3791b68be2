// partition_kernel.cuh — stable row-index partition after a split + per-tree preparation (sm_90a).
//
// Replaces: DataPartition::Split -> ParallelPartitionRunner::Run -> DenseBin::SplitInner
// (reference src/treelearner/data_partition.hpp:101-120, include/LightGBM/utils/threading.h:92-193,
// src/io/dense_bin.hpp:314-394), the child bookkeeping of SerialTreeLearner::SplitInner
// (src/treelearner/serial_tree_learner.cpp:769-925) and BeforeTrain/LeafSplits::Init (:291-341).
//
// Two launches per split, no host involvement:
//   k_part_flags   : go-left flag per row (decoded-bin form of SplitInner's 8 template cases) + per-block
//                    left counts.  Reads one byte per row straight from the row-major bin matrix.
//   k_part_scatter : every block re-derives its write offsets from the block counts, then writes the
//                    left rows followed by the right rows into the OTHER index buffer (ping-pong, so no
//                    copy-back pass as in the reference's two-buffer runner).  Stable in both halves.
//                    Thread 0 of block 0 then plays SplitInner: child leaf records, smaller/larger
//                    choice, histogram-slot hand-over, BeforeFindBestSplit gates, the split record.
#pragma once
#include "comm.cuh"
#include "types.cuh"

namespace b200 {

constexpr int kPartThreads = 256;

struct PartArgs {
  const uint8_t* bins;     // row-major [N x pitch] (used when no column-major copy exists)
  const uint8_t* binsT;    // column-major copy [Cpad x N] for the partition, or nullptr
  int64_t num_data;
  int64_t pitch;
  int32_t* idx0;
  int32_t* idx1;
  uint32_t* flag_words;    // [ceil(num_data/32)] bit-packed go-left flags (single GPU); feature-shard mode uses
                           // the CommBlock flag buffers instead
  int32_t* block_left;     // [gridDim.x]
  CommPeers peers;         // world == 1: plain local partition
  Leaf* leaves;
  Ctl* ctl;
  SplitRec* splits;        // [num_leaves-1] output records
  Params params;
  // leaf-ordered copies of the per-row fixed-point (g,h) [and of the packed quantized word], parallel to idx0 / idx1:
  // the scatter writes them next to the row ids, so that the histogram producers of a non-root leaf stream (g,h)
  // contiguously instead of gathering 8 bytes per row per column-group set (nullptr: off)
  const int2* gh; int2* gho0; int2* gho1;
  const int32_t* ghq; int32_t* ghqo0; int32_t* ghqo1;
};

// Decoded form of DenseBin::SplitInner (dense_bin.hpp:314-394): with b = the feature's bin of the row,
//   missing Zero & b == default_bin  -> default side
//   missing NaN  & b == num_bin - 1  -> default side
//   otherwise                        -> left iff b <= threshold
__device__ __forceinline__ bool goes_left(uint32_t v, const FeatMeta& m, int threshold, int default_left) {
  const int rel = static_cast<int>(v) - m.lo;
  const int b = (rel >= 0 && rel < m.nslice) ? rel + m.offset : m.mfb;
  if ((m.missing == 1 && b == m.default_bin) || (m.missing == 2 && b == m.num_bin - 1)) return default_left != 0;
  return b <= threshold;
}

__device__ __forceinline__ void part_block_range(int n, int nblocks, int b, int* lo, int* hi) {
  int per = (n + nblocks - 1) / nblocks;
  per = (per + kPartThreads - 1) / kPartThreads * kPartThreads;
  *lo = min(n, b * per);
  *hi = min(n, *lo + per);
}

// Go-left flags are BIT-packed, one 32-bit ballot word per 32 consecutive rows of the leaf (leaf-relative
// index i -> word i>>5, bit i&31).  Block ranges are multiples of 256 rows, so every warp owns whole words.
// Single GPU: words go to the local scratch.  Feature-shard: only the split's owner computes them and
// pushes them (and its per-block left counts) into every rank's CommBlock over NVLink (n/8 bytes per peer),
// then publishes a sequence number; k_part_scatter on every rank waits for it.
constexpr int kPartUnroll = 4;

__device__ __forceinline__ void part_flags_body(const PartArgs& a) {
  Ctl* c = a.ctl;
  if (!c->cur_valid) return;
  const int me = a.peers.rank;
  // row-shard: every rank flags its own rows; mode 2: every rank holds a copy of every partition column and
  // computes the flags of every split itself (no push, no wait)
  const int W = a.peers.mode == 0 ? a.peers.world : 1;
  if (W > 1 && c->cur_owner != me) return;        // feature-shard: only the rank that holds the split column computes flags
  const int n = c->cur_count, begin = c->cur_begin;
  const int32_t* src = (c->cur_buf ? a.idx1 : a.idx0) + begin;
  const FeatMeta m = c->cur_meta;
  const int threshold = c->cur_threshold, default_left = c->cur_default_left;
  const unsigned long long fseq = c->flag_seq;      // bumped by k_select when it chose this split
  const int par = static_cast<int>(fseq & 1);
  const int lane = threadIdx.x & 31;
  // the column-major copy turns the per-row 32-byte sector gather of the row-major matrix (1 useful byte per
  // sector, ~8x below DRAM peak at the root) into a near-sequential byte stream: rows of a leaf are ascending
  const bool use_t = a.binsT != nullptr;
  const uint8_t* colp = use_t ? a.binsT + static_cast<int64_t>(m.col) * a.num_data : a.bins + m.col;
  const int64_t rstride = use_t ? 1 : a.pitch;
  int lo, hi;
  part_block_range(n, gridDim.x, blockIdx.x, &lo, &hi);
  int cnt = 0;
  for (int base = lo; base < hi; base += kPartThreads * kPartUnroll) {
    // kPartUnroll independent (index -> bin byte) load chains per thread
    int row[kPartUnroll]; uint32_t v[kPartUnroll];
#pragma unroll
    for (int k = 0; k < kPartUnroll; ++k) {
      const int i = base + k * kPartThreads + threadIdx.x;
      row[k] = i < hi ? __ldg(src + i) : -1;
    }
#pragma unroll
    for (int k = 0; k < kPartUnroll; ++k) v[k] = row[k] >= 0 ? __ldg(colp + static_cast<int64_t>(row[k]) * rstride) : 0u;
#pragma unroll
    for (int k = 0; k < kPartUnroll; ++k) {
      const int i = base + k * kPartThreads + threadIdx.x;
      const bool left = row[k] >= 0 && goes_left(v[k], m, threshold, default_left);
      const unsigned word = __ballot_sync(0xffffffffu, left);
      if (lane == 0 && (i - lane) < hi) {
        const int wi = (i - lane) >> 5;
        if (W > 1) comm_flag_words(a.peers.block[me], par, a.peers.flags_stride)[wi] = word;   // own buffer first; pushed to the peers below
        else a.flag_words[wi] = word;
        cnt += __popc(word);
      }
    }
  }
  __shared__ int s_cnt[kPartThreads / 32];
  if (lane == 0) s_cnt[threadIdx.x >> 5] = cnt;
  __syncthreads();                         // also: this block's flag words (global) are visible block-wide
  int t = 0;
#pragma unroll
  for (int w = 0; w < kPartThreads / 32; ++w) t += s_cnt[w];
  if (W == 1) {
    if (threadIdx.x == 0) a.block_left[blockIdx.x] = t;
    return;
  }
  // feature-shard, owner: push this block's words (a contiguous, 32-byte aligned run) and its left count into
  // every rank's CommBlock with coalesced 16-byte peer stores over NVLink; the last block publishes the sequence
  // number.  Peers need no counting pass: k_part_scatter waits for the sequence number and reads blk_left.
  {
    const int w_lo = lo >> 5, w_hi = (hi + 31) >> 5;
    const uint4* src = reinterpret_cast<const uint4*>(comm_flag_words(a.peers.block[me], par, a.peers.flags_stride) + w_lo);
    const int nvec = lo < hi ? (w_hi - w_lo + 3) / 4 : 0;       // empty blocks (lo == hi == n) push nothing
    for (int i = threadIdx.x; i < nvec; i += kPartThreads) {
      const uint4 v = src[i];
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r) {
        if (r < W && r != me) reinterpret_cast<uint4*>(comm_flag_words(a.peers.block[r], par, a.peers.flags_stride) + w_lo)[i] = v;
      }
    }
    if (threadIdx.x < W) a.peers.block[threadIdx.x]->blk_left[par][blockIdx.x] = t;
    __threadfence_system();                // every thread orders its own peer stores
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned done = atomicAdd(&c->part_blocks_done, 1u);
      if (done == gridDim.x - 1) {
        __threadfence_system();
        for (int r = 0; r < W; ++r) st_release_sys(&a.peers.block[r]->flags_seq[par], fseq);
      }
    }
  }
}

__global__ void __launch_bounds__(kPartThreads) k_part_flags(const PartArgs a) {
  part_flags_body(a);
}

__device__ __forceinline__ void part_scatter_body(const PartArgs& a) {
  Ctl* c = a.ctl;
  if (!c->cur_valid) return;
  const int n = c->cur_count, begin = c->cur_begin;
  const int32_t* src = (c->cur_buf ? a.idx1 : a.idx0) + begin;
  int32_t* dst = (c->cur_buf ? a.idx0 : a.idx1) + begin;
  int2* gho = a.gho0 ? (c->cur_buf ? a.gho0 : a.gho1) + begin : nullptr;
  int32_t* ghqo = a.ghqo0 ? (c->cur_buf ? a.ghqo0 : a.ghqo1) + begin : nullptr;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t* fw = a.flag_words;
  const int32_t* block_left = a.block_left;
  if (a.peers.world > 1 && a.peers.mode == 0) {
    // feature-shard: the flag words and per-block counts of this split are pushed by the split's owner
    CommBlock* mine = a.peers.block[a.peers.rank];
    const int par = static_cast<int>(c->flag_seq & 1);
    __shared__ int s_ok;
    if (tid == 0) { s_ok = wait_seq(&mine->flags_seq[par], c->flag_seq) ? 1 : 0; if (!s_ok) c->error = 1; }
    __syncthreads();
    if (!s_ok) return;
    fw = comm_flag_words(mine, par, a.peers.flags_stride);
    block_left = mine->blk_left[par];
  }

  // offsets from the per-block counts (gridDim.x <= 1024)
  __shared__ int s_red[kPartUnroll][kPartThreads / 32];
  __shared__ int s_before, s_total;
  int before = 0, total = 0;
  for (int j = tid; j < static_cast<int>(gridDim.x); j += kPartThreads) {
    const int v = __ldcv(block_left + j);
    total += v;
    if (j < static_cast<int>(blockIdx.x)) before += v;
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) { total += __shfl_xor_sync(0xffffffffu, total, d); before += __shfl_xor_sync(0xffffffffu, before, d); }
  __shared__ int s_tot[kPartThreads / 32], s_bef[kPartThreads / 32];
  if (lane == 0) { s_tot[warp] = total; s_bef[warp] = before; }
  __syncthreads();
  if (tid == 0) {
    int t = 0, b = 0;
#pragma unroll
    for (int w = 0; w < kPartThreads / 32; ++w) { t += s_tot[w]; b += s_bef[w]; }
    s_total = t; s_before = b;
  }
  __syncthreads();
  const int total_left = s_total;
  int left_run = s_before;          // lefts before the current tile (whole leaf)
  // only the smaller child gets a histogram pass (the larger one is parent - smaller), so only its rows need the
  // leaf-ordered (g,h) copy; row-shard decides smaller/larger on GLOBAL counts after this kernel's exchange: copy both
  const bool copy_both = a.peers.world > 1 && a.peers.mode == 1;
  const bool left_smaller = total_left < n - total_left;        // same rule as the bookkeeping below (:858)

  int lo, hi;
  part_block_range(n, gridDim.x, blockIdx.x, &lo, &hi);
  for (int base = lo; base < hi; base += kPartThreads * kPartUnroll) {
    unsigned word[kPartUnroll]; int row[kPartUnroll];
    int2 gv[kPartUnroll]; int qv[kPartUnroll];
#pragma unroll
    for (int k = 0; k < kPartUnroll; ++k) {
      const int i = base + k * kPartThreads + tid;
      const int w0 = i - lane;                       // first row of this warp's word
      word[k] = (w0 < hi) ? __ldcv(fw + (w0 >> 5)) : 0u;
      row[k] = (i < hi) ? src[i] : -1;
      if (lane == 0) s_red[k][warp] = __popc(word[k]);
    }
#pragma unroll
    for (int k = 0; k < kPartUnroll; ++k) {
      const bool mine = copy_both || ((((word[k] >> lane) & 1u) != 0u) == left_smaller);
      gv[k] = (gho != nullptr && row[k] >= 0 && mine) ? __ldg(a.gh + row[k]) : make_int2(0, 0);
      qv[k] = (ghqo != nullptr && row[k] >= 0 && mine) ? __ldg(a.ghq + row[k]) : 0;
    }
    __syncthreads();
    int run = left_run;
#pragma unroll
    for (int k = 0; k < kPartUnroll; ++k) {
      int wbefore = 0, tile_left = 0;
#pragma unroll
      for (int w = 0; w < kPartThreads / 32; ++w) { const int v = s_red[k][w]; if (w < warp) wbefore += v; tile_left += v; }
      const int i = base + k * kPartThreads + tid;
      if (i < hi) {
        const int lefts_before_me = run + wbefore + __popc(word[k] & ((1u << lane) - 1u));
        const int pos = ((word[k] >> lane) & 1u) ? lefts_before_me : total_left + (i - lefts_before_me);
        dst[pos] = row[k];
        const bool mine = copy_both || ((((word[k] >> lane) & 1u) != 0u) == left_smaller);
        if (gho != nullptr && mine) gho[pos] = gv[k];
        if (ghqo != nullptr && mine) ghqo[pos] = qv[k];
      }
      run += tile_left;
    }
    left_run = run;
    __syncthreads();
  }

  // ---- SplitInner bookkeeping: serial_tree_learner.cpp:769-925, tree.h:543-585
  // row-shard: the children's GLOBAL row counts decide smaller/larger and the min-data gates; block 0 all-gathers
  // the local left/right counts first (DataParallelTreeLearner keeps global_data_count_in_leaf_ the same way,
  // reference src/treelearner/data_parallel_tree_learner.cpp:254-262)
  if (blockIdx.x != 0) return;
  __shared__ double s_in[8];
  __shared__ double s_out[kMaxRanks][8];
  int g_left = total_left, g_right = n - total_left;
  if (a.peers.world > 1 && a.peers.mode == 1) {
    if (tid == 0) { s_in[0] = total_left; s_in[1] = n - total_left; for (int k = 2; k < 8; ++k) s_in[k] = 0; }
    __syncthreads();
    exchange_misc(a.peers, c, s_in, s_out);
    g_left = 0; g_right = 0;
    for (int r = 0; r < a.peers.world; ++r) { g_left += static_cast<int>(s_out[r][0]); g_right += static_cast<int>(s_out[r][1]); }
  }
  if (tid == 0) {
    const int leaf = c->cur_leaf;
    const int right = c->num_leaves;          // next_leaf_id
    Leaf& L = a.leaves[leaf];
    Leaf& R = a.leaves[right];
    const Cand s = L.best;
    const int left_count = g_left, right_count = g_right;          // global
    const int lleft = total_left, lright = n - total_left;         // this rank's rows
    SplitRec& rec = a.splits[right - 1];
    rec.leaf = leaf; rec.feature = s.feature; rec.threshold = s.threshold; rec.default_left = s.default_left;
    rec.left_count = left_count; rec.right_count = right_count; rec.owner = s.owner; rec.pad = 0;
    rec.gain = s.gain; rec.lsg = s.lsg; rec.lsh = s.lsh; rec.lout = s.lout; rec.rsg = s.rsg; rec.rsh = s.rsh; rec.rout = s.rout;

    const int parent_slot = L.slot, parent_depth = L.depth, child_buf = 1 - L.buf;
    R.begin = begin + lleft; R.count = right_count; R.lcount = lright; R.buf = child_buf; R.depth = parent_depth + 1;
    R.sum_g = s.rsg; R.sum_h = s.rsh; R.output = s.rout;
    R.best.gain = -INFINITY; R.best.feature = -1; R.best.real = 0x7fffffff; R.best.owner = 0;
    L.count = left_count; L.lcount = lleft; L.buf = child_buf; L.depth = parent_depth + 1;
    // quantized training: SplitInfo::{left,right}_sum_gradient_and_hessian -> LeafSplits::Init (serial_tree_learner.cpp:880-905)
    R.isum_g = L.isum_g - s.ilg; R.isum_h = L.isum_h - s.ilh;
    L.isum_g = s.ilg; L.isum_h = s.ilh;
    L.sum_g = s.lsg; L.sum_h = s.lsh; L.output = s.lout;
    L.best.gain = -INFINITY; L.best.feature = -1; L.best.real = 0x7fffffff; L.best.owner = 0;
    // smaller / larger (serial_tree_learner.cpp:858): the parent's pool slot becomes the larger child's,
    // the smaller child gets the fresh slot `right` (one new slot per split, zeroed at the start of the tree)
    int smaller, larger;
    if (left_count < right_count) { smaller = leaf; larger = right; } else { smaller = right; larger = leaf; }
    a.leaves[larger].slot = parent_slot;
    a.leaves[smaller].slot = right;
    c->smaller = smaller; c->larger = larger;
    c->num_leaves = right + 1;
    // BeforeFindBestSplit (serial_tree_learner.cpp:343-370)
    int do_find = 1;
    if (a.params.max_depth > 0 && parent_depth + 1 >= a.params.max_depth) do_find = 0;
    if (right_count < a.params.min_data_in_leaf * 2 && left_count < a.params.min_data_in_leaf * 2) do_find = 0;
    c->do_find = do_find;
    if (c->error) c->cur_valid = 0;
  }
}

__global__ void __launch_bounds__(kPartThreads) k_part_scatter(const PartArgs a) {
  part_scatter_body(a);
}

// One-off at Init: column-major copy of the bin matrix (32x32 byte tiles through shared memory)
__global__ void __launch_bounds__(256) k_transpose_bins(const uint8_t* __restrict__ bins, int64_t pitch, int64_t N, int C,
                                                        uint8_t* __restrict__ binsT) {
  __shared__ uint8_t tile[32][33];
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8 threads
  for (int j = ty; j < 32; j += 8) {
    const int64_t r = r0 + j;
    tile[j][tx] = (r < N && c0 + tx < C) ? bins[r * pitch + c0 + tx] : 0;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const int64_t r = r0 + tx;
    if (c < C && r < N) binsT[static_cast<int64_t>(c) * N + r] = tile[tx][j];
  }
}

// ---------------------------------------------------------------------------------------------------
// Per-tree preparation: pack (grad,hess), identity index list, root sums (BeforeTrain).
struct PrepArgs {
  const float* grad;
  const float* hess;
  int2* gq;                 // [num_data] fixed-point (g, h) of this tree (k_quant_rows; quantized training: k_quantize)
  int32_t* idx0;
  const int32_t* bag;       // device bag indices or nullptr
  const int32_t* bag_count; // device: number of bag indices (read by the kernels, so that a new bag of a different size —
                            // bagging or GOSS every iteration — replays the SAME captured graph)
  int32_t num_data;
  PartialSum* partials;     // [gridDim.x]
  Leaf* leaves;
  Ctl* ctl;
  Params params;
  int32_t max_leaves;
  int32_t num_partials;
  CommPeers peers;
  int32_t* ghq;             // quantized training: packed (g << 16) + h per row for k_hist_q, or nullptr
};

constexpr int kPrepThreads = 256;

__global__ void __launch_bounds__(kPrepThreads) k_prep(const PrepArgs a) {
  // fixed block -> row-range assignment and a fixed-order final reduction => deterministic root sums
  const int N = a.num_data;
  const int nb = gridDim.x;
  int per = (N + nb - 1) / nb;
  per = (per + kPrepThreads - 1) / kPrepThreads * kPrepThreads;
  const int lo = min(N, static_cast<int>(blockIdx.x) * per), hi = min(N, lo + per);
  double sg = 0.0, sh = 0.0; float mg = 0.f, mh = 0.f;
  for (int i = lo + threadIdx.x; i < hi; i += kPrepThreads) {
    const float g = a.grad[i], h = a.hess[i];
    mg = fmaxf(mg, fabsf(g)); mh = fmaxf(mh, fabsf(h));
    if (a.bag == nullptr) { sg += g; sh += h; a.idx0[i] = i; }
  }
  if (a.bag != nullptr) {
    const int bag_n = *a.bag_count;
    int perb = (bag_n + nb - 1) / nb;
    perb = (perb + kPrepThreads - 1) / kPrepThreads * kPrepThreads;
    const int blo = min(bag_n, static_cast<int>(blockIdx.x) * perb), bhi = min(bag_n, blo + perb);
    for (int i = blo + threadIdx.x; i < bhi; i += kPrepThreads) {
      const int r = a.bag[i];
      a.idx0[i] = r;
      sg += a.grad[r]; sh += a.hess[r];
    }
  }
  __shared__ double s_g[kPrepThreads / 32], s_h[kPrepThreads / 32];
  __shared__ float s_mg[kPrepThreads / 32], s_mh[kPrepThreads / 32];
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    sg += __shfl_xor_sync(0xffffffffu, sg, d); sh += __shfl_xor_sync(0xffffffffu, sh, d);
    mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, d)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, d));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_g[warp] = sg; s_h[warp] = sh; s_mg[warp] = mg; s_mh[warp] = mh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    PartialSum p; p.g = 0; p.h = 0; p.gmax = 0; p.hmax = 0;
    for (int w = 0; w < kPrepThreads / 32; ++w) { p.g += s_g[w]; p.h += s_h[w]; p.gmax = fmaxf(p.gmax, s_mg[w]); p.hmax = fmaxf(p.hmax, s_mh[w]); }
    a.partials[blockIdx.x] = p;
  }
}

__device__ __forceinline__ double pow2_scale(double bound) {
  // largest power of two s with bound * s < 2^30 (bound = max|value| over the rows): every row's value becomes a
  // 30-bit integer (hist_atom_kernel.cuh), and a sum over up to 2^31 rows stays below 2^61
  if (!(bound > 0.0)) return 1.0;
  int e; frexp(bound, &e);            // bound < 2^e
  int k = 30 - e;
  if (k > 1000) k = 1000;
  if (k < -1000) k = -1000;
  return ldexp(1.0, k);
}

__global__ void __launch_bounds__(32) k_root_init(const PrepArgs a) {
  __shared__ double s_in[8];
  __shared__ double s_out[kMaxRanks][8];
  const int tid = threadIdx.x;
  const bool rows = a.peers.world > 1 && a.peers.mode == 1;
  if (tid == 0) {
    double sg = 0.0, sh = 0.0; float mg = 0.f, mh = 0.f;
    for (int b = 0; b < a.num_partials; ++b) { sg += a.partials[b].g; sh += a.partials[b].h; mg = fmaxf(mg, a.partials[b].gmax); mh = fmaxf(mh, a.partials[b].hmax); }
    s_in[0] = sg; s_in[1] = sh; s_in[2] = mg; s_in[3] = mh; s_in[4] = a.bag ? *a.bag_count : a.num_data;
    s_in[5] = s_in[6] = s_in[7] = 0;
  }
  __syncthreads();
  if (rows) {
    // row-shard: LeafSplits::Init sums are global (cuda_leaf_splits.cu:337-340 all-reduces them with NCCL;
    // here: all-gather over peer memory + a fixed-order sum => bitwise identical on every rank)
    exchange_misc(a.peers, a.ctl, s_in, s_out);
  }
  if (tid != 0) return;
  double sg = s_in[0], sh = s_in[1]; float mg = static_cast<float>(s_in[2]), mh = static_cast<float>(s_in[3]);
  const int n_local = static_cast<int>(s_in[4]);
  int n_root = n_local;
  if (rows) {
    sg = 0; sh = 0; mg = 0; mh = 0; n_root = 0;
    for (int r = 0; r < a.peers.world; ++r) {
      sg += s_out[r][0]; sh += s_out[r][1];
      mg = fmaxf(mg, static_cast<float>(s_out[r][2])); mh = fmaxf(mh, static_cast<float>(s_out[r][3]));
      n_root += static_cast<int>(s_out[r][4]);
    }
  }
  for (int i = 0; i < a.max_leaves; ++i) {
    Leaf& L = a.leaves[i];
    L.begin = 0; L.count = 0; L.buf = 0; L.depth = 0; L.slot = 0; L.lcount = 0;
    L.sum_g = 0; L.sum_h = 0; L.output = 0; L.isum_g = 0; L.isum_h = 0;
    L.best.gain = -INFINITY; L.best.feature = -1; L.best.real = 0x7fffffff; L.best.owner = 0;
  }
  Leaf& R = a.leaves[0];
  Ctl* c = a.ctl;
  long long isg = 0, ish = 0;
  if (a.params.quant) {
    // k_quantize left the INTEGER root sums in the partials (exact in fp64).  LeafSplits::Init(int8 ...)
    // (leaf_splits.hpp:117-140): sum_gradients_ = sum(int * scale); here int_sum * scale (one rounding).
    isg = __double2ll_rn(sg); ish = __double2ll_rn(sh);
    sg = static_cast<double>(isg) * c->q_gscale; sh = static_cast<double>(ish) * c->q_hscale;
  }
  R.isum_g = isg; R.isum_h = ish;
  R.count = n_root; R.lcount = n_local; R.sum_g = sg; R.sum_h = sh;
  // root output (serial_tree_learner.cpp:207-211): L1 + max_delta_step, no smoothing
  {
    double ret = -sg;
    if (a.params.l1 > 0.0) { double r = fabs(sg) - a.params.l1; if (r < 0) r = 0; ret = -((sg > 0) - (sg < 0)) * r; }
    ret /= (sh + a.params.l2);
    if (a.params.max_delta_step > 0 && fabs(ret) > a.params.max_delta_step) ret = ((ret > 0) - (ret < 0)) * a.params.max_delta_step;
    R.output = ret;
  }
  c->cur_valid = c->error ? 0 : 1; c->cur_owner = 0; c->part_blocks_done = 0; c->cur_leaf = 0; c->cur_begin = 0; c->cur_count = n_local; c->cur_buf = 0;
  c->smaller = 0; c->larger = -1; c->do_find = 1; c->num_leaves = 1;
  // BeforeFindBestSplit at the root: too few rows to ever split
  if (n_root < a.params.min_data_in_leaf * 2) c->do_find = 0;
  c->g_scale = pow2_scale(static_cast<double>(mg));
  c->h_scale = pow2_scale(static_cast<double>(mh));
  if (a.params.quant) { c->g_scale = 1.0; c->h_scale = 1.0; }     // the pool holds the raw integer sums
  c->g_inv = 1.0 / c->g_scale; c->h_inv = 1.0 / c->h_scale;
  c->root_sum_g = sg; c->root_sum_h = sh; c->root_count = n_root; c->root_identity = a.bag ? 0 : 1;
  // constant hessian (Init(..., is_constant_hessian)): the per-row fixed-point hessian the histogram kernel scales its
  // row counts with (the reference counts and multiplies by hessians[0] the same way, dataset.cpp:1430-1437)
  c->h_const_q = a.params.quant ? 1 : llrint(static_cast<double>(a.hess[0]) * c->h_scale);
}

// Per-tree fixed point: q = rint(value * scale), scale = the power of two k_root_init just chose (|q| < 2^30).
__global__ void __launch_bounds__(kPrepThreads) k_quant_rows(const PrepArgs a) {
  const Ctl* c = a.ctl;
  const double gs = c->g_scale, hs = c->h_scale;       // powers of two: the products are exact, one rounding to integer
  for (int i = blockIdx.x * kPrepThreads + threadIdx.x; i < a.num_data; i += gridDim.x * kPrepThreads)
    a.gq[i] = make_int2(__double2int_rn(static_cast<double>(a.grad[i]) * gs), __double2int_rn(static_cast<double>(a.hess[i]) * hs));
}

// ---- quantized-gradient training: GradientDiscretizer::DiscretizeGradients (gradient_discretizer.cpp:68-160) ----
// k_prep has left max|g|, max|h| over ALL rows in the partials.  k_quant_scales turns them into the tree's scales;
// k_quantize writes the int8 values into gq[] (consumed by
// k_hist<true>) and replaces the partials by the integer root sums (over the bag if there is one).
__global__ void __launch_bounds__(32) k_quant_scales(const PrepArgs a) {
  if (threadIdx.x != 0) return;
  float mg = 0.f, mh = 0.f;
  for (int b = 0; b < a.num_partials; ++b) { mg = fmaxf(mg, a.partials[b].gmax); mh = fmaxf(mh, a.partials[b].hmax); }
  Ctl* c = a.ctl;
  const double max_g = mg, max_h = mh;
  c->q_gscale = max_g / static_cast<double>(a.params.quant_bins / 2);
  c->q_hscale = a.params.quant_const_hess ? max_h : max_h / static_cast<double>(a.params.quant_bins);
  // the reference divides the float literal 1.0f by the double scale; all-zero gradients (scale 0) would make that
  // inf and the discretized values NaN casts: map them to 0 instead (no split is found, as it should be)
  c->q_ginv = c->q_gscale > 0.0 ? 1.0f / c->q_gscale : 0.0;
  c->q_hinv = c->q_hscale > 0.0 ? 1.0f / c->q_hscale : 0.0;
  c->quant_iter += 1;
}

// counter-based uniform in [0,1) (splitmix64 finaliser over (seed, tree, row, stream)).  The counter is
// row << 1 | stream: stochastic rounding draws on streams 0 and 1, which fill bit 0.  Rows are below 2^31, so those
// counters stay below 2^32, and GOSS draws on kGossStream, the bit above them: every (row, stream) has its own counter.
constexpr unsigned long long kGossStream = 1ull << 32;
__device__ __forceinline__ double quant_uniform(unsigned long long seed, unsigned long long iter, unsigned row, unsigned long long stream) {
  unsigned long long z = seed * 0x9E3779B97F4A7C15ull + iter * 0xBF58476D1CE4E5B9ull + (static_cast<unsigned long long>(row) << 1 | stream);
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return static_cast<double>(z >> 11) * (1.0 / 9007199254740992.0);
}

__device__ __forceinline__ int2 quantize_row(const PrepArgs& a, const Ctl* c, int i) {
  const double g = a.grad[i];
  double rg = 0.5, rh = 0.5;
  if (a.params.quant_stochastic) {
    rg = quant_uniform(static_cast<unsigned>(a.params.quant_seed), c->quant_iter, static_cast<unsigned>(i), 0u);
    rh = quant_uniform(static_cast<unsigned>(a.params.quant_seed), c->quant_iter, static_cast<unsigned>(i), 1u);
  }
  // static_cast<int8_t>(double): truncation toward zero (gradient_discretizer.cpp:123-125, :146-148)
  const int qg = g >= 0.0 ? static_cast<int>(g * c->q_ginv + rg) : static_cast<int>(g * c->q_ginv - rg);
  const int qh = a.params.quant_const_hess ? 1 : static_cast<int>(static_cast<double>(a.hess[i]) * c->q_hinv + rh);
  return make_int2(static_cast<int>(static_cast<signed char>(qg)), static_cast<int>(static_cast<signed char>(qh)));
}

__global__ void __launch_bounds__(kPrepThreads) k_quantize(const PrepArgs a) {
  const Ctl* c = a.ctl;
  const int N = a.num_data;
  const int nb = gridDim.x;
  int per = (N + nb - 1) / nb;
  per = (per + kPrepThreads - 1) / kPrepThreads * kPrepThreads;
  const int lo = min(N, static_cast<int>(blockIdx.x) * per), hi = min(N, lo + per);
  long long sg = 0, sh = 0; int mg = 0, mh = 0;
  for (int i = lo + threadIdx.x; i < hi; i += kPrepThreads) {
    const int2 q = quantize_row(a, c, i);
    a.gq[i] = q;
    if (a.ghq != nullptr) a.ghq[i] = q.x * 65536 + q.y;
    mg = max(mg, abs(q.x)); mh = max(mh, abs(q.y));
    if (a.bag == nullptr) { sg += q.x; sh += q.y; }
  }
  if (a.bag != nullptr) {
    const int bag_n = *a.bag_count;
    int perb = (bag_n + nb - 1) / nb;
    perb = (perb + kPrepThreads - 1) / kPrepThreads * kPrepThreads;
    const int blo = min(bag_n, static_cast<int>(blockIdx.x) * perb), bhi = min(bag_n, blo + perb);
    for (int i = blo + threadIdx.x; i < bhi; i += kPrepThreads) {
      const int2 q = quantize_row(a, c, a.bag[i]);       // recomputed: the row may belong to another block's range
      sg += q.x; sh += q.y;
    }
  }
  __shared__ long long s_g[kPrepThreads / 32], s_h[kPrepThreads / 32];
  __shared__ int s_mg[kPrepThreads / 32], s_mh[kPrepThreads / 32];
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    sg += __shfl_xor_sync(0xffffffffu, sg, d); sh += __shfl_xor_sync(0xffffffffu, sh, d);
    mg = max(mg, __shfl_xor_sync(0xffffffffu, mg, d)); mh = max(mh, __shfl_xor_sync(0xffffffffu, mh, d));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_g[warp] = sg; s_h[warp] = sh; s_mg[warp] = mg; s_mh[warp] = mh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long tg = 0, th = 0; int tmg = 0, tmh = 0;
    for (int w = 0; w < kPrepThreads / 32; ++w) { tg += s_g[w]; th += s_h[w]; tmg = max(tmg, s_mg[w]); tmh = max(tmh, s_mh[w]); }
    PartialSum p; p.g = static_cast<double>(tg); p.h = static_cast<double>(th); p.gmax = static_cast<float>(tmg); p.hmax = static_cast<float>(tmh);
    a.partials[blockIdx.x] = p;
  }
}

// Config::quant_train_renew_leaf — GradientDiscretizer::RenewIntGradTreeOutput (gradient_discretizer.cpp:236-259):
// leaf outputs from the ORIGINAL gradients of the leaf's rows, <USE_L1, USE_MAX_OUTPUT, no smoothing>, parent_output 0.
// Pass 1: per-(leaf, block) partial sums in a fixed order; pass 2 (k_renew_leaf_finish): fixed-order total + output.
struct RenewArgs {
  const float* grad; const float* hess;
  const Leaf* leaves; const Ctl* ctl;
  const int32_t* idx0; const int32_t* idx1;
  double* partial;          // [max_leaves][gridDim.x][2]
  double* out;              // [max_leaves]
  Params params;
};
__global__ void __launch_bounds__(256) k_renew_leaf(const RenewArgs a) {
  const int leaf = blockIdx.y;
  double sg = 0.0, sh = 0.0;
  if (leaf < a.ctl->num_leaves) {
    const Leaf& L = a.leaves[leaf];
    const int32_t* idx = (L.buf ? a.idx1 : a.idx0) + L.begin;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < L.lcount; i += gridDim.x * 256) {
      const int r = idx[i];
      sg += a.grad[r]; sh += a.hess[r];
    }
  }
  __shared__ double s_g[8], s_h[8];
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) { sg += __shfl_xor_sync(0xffffffffu, sg, d); sh += __shfl_xor_sync(0xffffffffu, sh, d); }
  if ((threadIdx.x & 31) == 0) { s_g[threadIdx.x >> 5] = sg; s_h[threadIdx.x >> 5] = sh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double tg = 0, th = 0;
    for (int w = 0; w < 8; ++w) { tg += s_g[w]; th += s_h[w]; }
    double* p = a.partial + (static_cast<int64_t>(leaf) * gridDim.x + blockIdx.x) * 2;
    p[0] = tg; p[1] = th;
  }
}
__global__ void k_renew_leaf_finish(const RenewArgs a, int blocks) {
  const int leaf = blockIdx.x * blockDim.x + threadIdx.x;
  if (leaf >= a.params.num_leaves) return;
  if (leaf >= a.ctl->num_leaves) { a.out[leaf] = 0.0; return; }
  double sg = 0.0, sh = 0.0;
  for (int b = 0; b < blocks; ++b) { const double* p = a.partial + (static_cast<int64_t>(leaf) * blocks + b) * 2; sg += p[0]; sh += p[1]; }
  double ret = -sg;
  if (a.params.l1 > 0.0) { double r = fabs(sg) - a.params.l1; if (r < 0) r = 0; ret = -((sg > 0) - (sg < 0)) * r; }
  ret /= (sh + a.params.l2);
  if (a.params.max_delta_step > 0 && fabs(ret) > a.params.max_delta_step) ret = ((ret > 0) - (ret < 0)) * a.params.max_delta_step;
  a.out[leaf] = ret;
}

// row-shard: tell every peer that this rank's local histogram for the current iteration is complete
// (launched right after k_hist: stream order guarantees the REDs have been performed)
__global__ void __launch_bounds__(32) k_hist_signal(const CommPeers peers, Ctl* c) {
  if (!c->cur_valid || !c->do_find) return;
  const unsigned long long seq = c->hist_seq + 1;
  if (threadIdx.x < peers.world) {
    __threadfence_system();
    st_release_sys(&peers.block[threadIdx.x]->hist_seq[peers.rank], seq);
  }
  __syncwarp();
  if (threadIdx.x == 0) c->hist_seq = seq;
}

// AddPredictionToScore (serial_tree_learner.h:100-115): one grid row per leaf
struct ScoreArgs {
  const Leaf* leaves;
  const int32_t* idx0;
  const int32_t* idx1;
  const double* leaf_value;   // device [num_leaves]
  double* score;
};

__global__ void __launch_bounds__(256) k_add_score(const ScoreArgs a) {
  const Leaf& L = a.leaves[blockIdx.y];
  const int32_t* idx = (L.buf ? a.idx1 : a.idx0) + L.begin;
  const double v = a.leaf_value[blockIdx.y];
  for (int i = blockIdx.x * 256 + threadIdx.x; i < L.lcount; i += gridDim.x * 256) a.score[idx[i]] += v;
}

// row -> leaf id of the final partition (one grid row per leaf)
template <typename T>
__global__ void __launch_bounds__(256) k_leaf_index(const Leaf* leaves, const int32_t* idx0, const int32_t* idx1, T* row_leaf) {
  const Leaf& L = leaves[blockIdx.y];
  const int32_t* idx = (L.buf ? idx1 : idx0) + L.begin;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < L.lcount; i += gridDim.x * 256) row_leaf[idx[i]] = static_cast<T>(blockIdx.y);
}

// Route EVERY row through the tree that was just grown (the split records in application order) and add its leaf's
// value to the score / record its leaf id.  With a bagging set (bagging, GOSS) the partition only holds the bagged
// rows; the reference scores the out-of-bag rows by predicting the tree on them (GBDT::UpdateScore, gbdt.cpp:505-530 ->
// Tree::AddPredictionToScore on bin iterators): this is that, over the device bin matrix, replaying the splits:
// a row sitting in leaf s.leaf when split i is applied moves to leaf i + 1 iff it does not go left.
struct RouteSplit { int32_t leaf, col, threshold, default_left; FeatMeta m; };
constexpr int kRouteMaxSplits = 1024;
__global__ void __launch_bounds__(256) k_route_rows(const uint8_t* __restrict__ bins, int64_t pitch, int n, const SplitRec* splits,
                                                    const FeatMeta* feat, int num_splits, const double* leaf_value, double* score,
                                                    int32_t* row_leaf) {
  extern __shared__ RouteSplit s_sp[];
  for (int i = threadIdx.x; i < num_splits; i += blockDim.x) {
    const SplitRec r = splits[i];
    RouteSplit q; q.leaf = r.leaf; q.m = feat[r.feature]; q.col = q.m.col; q.threshold = r.threshold; q.default_left = r.default_left;
    s_sp[i] = q;
  }
  __syncthreads();
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < n; row += gridDim.x * blockDim.x) {
    const uint8_t* rp = bins + static_cast<int64_t>(row) * pitch;
    int leaf = 0;
    for (int i = 0; i < num_splits; ++i) {
      const RouteSplit& q = s_sp[i];
      if (q.leaf == leaf && !goes_left(rp[q.col], q.m, q.threshold, q.default_left)) leaf = i + 1;
    }
    if (score != nullptr) score[row] += leaf_value[leaf];
    if (row_leaf != nullptr) row_leaf[row] = leaf;
  }
}

__global__ void k_fill_f32(float* p, float v, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = v;
}

// L2 objective gradients (regression_objective.hpp:127-142, unweighted): g = score - label, h = 1
__global__ void k_l2_gradients(const double* score, const float* label, float* grad, float* hess, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    grad[i] = static_cast<float>(score[i] - label[i]);
    hess[i] = 1.0f;
  }
}

// Binary logloss gradients (binary_objective.hpp:105-121, unweighted, label_weights = 1): label in {0,1}
__global__ void k_binary_gradients(const double* score, const float* label, float* grad, float* hess, int n, double sigmoid) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int lab = label[i] > 0.0f ? 1 : -1;
    const double response = -lab * sigmoid / (1.0 + exp(lab * sigmoid * score[i]));
    const double abs_response = fabs(response);
    grad[i] = static_cast<float>(response);
    hess[i] = static_cast<float>(abs_response * (sigmoid - abs_response));
  }
}

}  // namespace b200
