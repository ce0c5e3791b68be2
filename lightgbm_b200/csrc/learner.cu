// learner.cu — host runtime + C-ABI of the tree learner (see include/lgbm_b200.h).
//
// Host side of SerialTreeLearner::Train (reference src/treelearner/serial_tree_learner.cpp:182-248)
// re-thought for a GPU that must not wait for the host: the leaf-wise loop is a FIXED launch sequence
//   prep, root_init, memset splittable, memset block counters, hist, scan, select      (root)
//   { part_flags, part_scatter, hist, scan, select } x (num_leaves-2), part_flags, part_scatter
// (hist = k_hist_a + k_hist_reduce, which overwrite their pool slot; the packed-cell k_hist_q of quantized training adds
// into it, so there the second memset zeroes the pool instead) whose every data-dependent decision (which leaf, which
// feature/threshold, smaller/larger child, early stop) is taken on the device through the Ctl block.  The sequence is
// captured once into a CUDA graph and replayed per tree; the host synchronises exactly once per tree, to read the split
// records back.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <cstdlib>
#include <vector>

#include "../../include/lgbm_b200.h"
#include "hist_atom_kernel.cuh"
#include "hist_q_kernel.cuh"
#include "goss_kernel.cuh"
#include "partition_kernel.cuh"
#include "scan_kernel.cuh"
#include "types.cuh"

namespace b200 {

static thread_local std::string g_last_error = "everything is fine";

struct CudaError {
  std::string msg;
};

#define CUDA_CHECK(expr)                                                                              \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) {                                                                          \
      char _buf[512];                                                                                 \
      snprintf(_buf, sizeof(_buf), "CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, \
               cudaGetErrorString(_e));                                                               \
      throw CudaError{_buf};                                                                          \
    }                                                                                                 \
  } while (0)

#define REQUIRE(cond, msg)                        \
  do {                                            \
    if (!(cond)) throw CudaError{std::string(msg)}; \
  } while (0)

// SM count of `device`; the sm_90a cubin (the only code in this library) loads on compute capability 9.0 alone
static int DeviceSms(int device) {
  int major = 0, minor = 0, sms = 0;
  CUDA_CHECK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CUDA_CHECK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  REQUIRE(major == 9 && minor == 0, "lgbm_b200 kernels are built for sm_90a (Hopper, H100) only");
  CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  return sms;
}

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  void alloc(size_t count) {
    release();
    if (count == 0) count = 1;
    CUDA_CHECK(cudaMalloc(&p, count * sizeof(T)));
    n = count;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr; n = 0;
  }
  ~DevBuf() { release(); }
};

// (re)allocate `d` to the size of `h` and copy `h` into it
template <typename T>
static void Up(DevBuf<T>& d, const std::vector<T>& h) {
  d.alloc(h.size());
  if (!h.empty()) CUDA_CHECK(cudaMemcpy(d.p, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice));
}

class Learner {
 public:
  explicit Learner(const LGBMB200_Config& cfg) { SetConfig(cfg); }
  ~Learner() { Destroy(); }

  // Developer A/B switches (not part of the boundary): LGBMB200_DEBUG is a bit mask read once per process.
  //   2: no TMA staging   64: quantized training never uses the packed-cell kernel   256: no leaf-ordered (g,h) copies
  // Each forces a path that also runs without it (the TMA-less fallback, quantized training with more than 15 bins, the
  // gathered stand-alone histogram hook), and tests/test_gpu_hist_exact.py requires the same bits as the default from it,
  // as from LGBMB200_SPLIT_K.  LGBMB200_PF and LGBMB200_PRED_PASS tune a parameter of the shipped kernels.
  static int DebugBits() {
    static const int bits = std::getenv("LGBMB200_DEBUG") ? std::atoi(std::getenv("LGBMB200_DEBUG")) : 0;
    return bits;
  }

  void SetConfig(const LGBMB200_Config& cfg) {
    REQUIRE(cfg.num_leaves >= 2, "num_leaves must be >= 2");
    const bool leaves_changed = cfg.num_leaves != cfg_.num_leaves || (cfg.use_quantized_grad != 0) != (params_.quant != 0);
    cfg_ = cfg;
    params_.num_leaves = cfg.num_leaves; params_.max_depth = cfg.max_depth; params_.min_data_in_leaf = cfg.min_data_in_leaf;
    params_.pad = 0;
    params_.min_sum_hessian = cfg.min_sum_hessian_in_leaf; params_.l1 = cfg.lambda_l1; params_.l2 = cfg.lambda_l2;
    params_.min_gain_to_split = cfg.min_gain_to_split; params_.max_delta_step = cfg.max_delta_step;
    params_.path_smooth = cfg.path_smooth;
    params_.quant = cfg.use_quantized_grad ? 1 : 0;
    params_.quant_bins = cfg.num_grad_quant_bins;
    params_.quant_renew = cfg.quant_train_renew_leaf ? 1 : 0;
    params_.quant_stochastic = cfg.stochastic_rounding ? 1 : 0;
    params_.quant_const_hess = const_hess_ ? 1 : 0;
    params_.quant_seed = cfg.seed;
    if (params_.quant && inited_ && ghq_.n < static_cast<size_t>(N_)) { ghq_.alloc(N_); ghqo0_.alloc(N_); ghqo1_.alloc(N_); }
    if (params_.quant) {
      REQUIRE(cfg.num_grad_quant_bins >= 2 && cfg.num_grad_quant_bins <= 127, "num_grad_quant_bins must be in [2, 127] (int8 gradients)");
      REQUIRE(!(peers_.world > 1 && peers_.mode == 1), "use_quantized_grad is not supported in row-shard mode");
    }
    InvalidateGraph();
    if (inited_ && leaves_changed) AllocTreeState();
  }

  void Init(const LGBMB200_Layout& lay, const uint8_t* bins_host, int is_constant_hessian) {
    REQUIRE(lay.num_data > 0 && lay.num_columns > 0 && lay.num_features > 0, "empty dataset");
    if (cfg_.gpu_device_id >= 0) { CUDA_CHECK(cudaSetDevice(cfg_.gpu_device_id)); }
    CUDA_CHECK(cudaGetDevice(&device_));
    num_sms_ = DeviceSms(device_);
    if (!stream_) CUDA_CHECK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    InvalidateGraph();

    N_ = lay.num_data; C_ = lay.num_columns; F_ = lay.num_features;
    Cpad_ = (C_ + 2 * kColGroup - 1) / (2 * kColGroup) * (2 * kColGroup);     // whole column-group PAIRS: 64-byte rows = whole DRAM atoms
    pitch_ = Cpad_;
    std::vector<FeatMeta> fm(F_);
    for (int f = 0; f < F_; ++f) {
      FeatMeta& m = fm[f];
      m.col = lay.feat_column[f]; m.lo = lay.feat_lo[f]; m.num_bin = lay.feat_num_bin[f];
      m.mfb = lay.feat_most_freq_bin[f]; m.offset = (m.mfb == 0) ? 1 : 0; m.nslice = m.num_bin - m.offset;
      m.default_bin = lay.feat_default_bin[f]; m.missing = lay.feat_missing_type[f]; m.real_index = lay.feat_real_index[f];
      REQUIRE(m.col >= 0 && m.col < C_, "feature column out of range");
      REQUIRE(m.num_bin >= 1 && m.lo >= 0 && m.lo + m.nslice <= kBinsPerColumn,
              "feature histogram slice exceeds 256 stored values per column (max_bin > 255 is not supported)");
    }
    feat_.alloc(F_);
    CUDA_CHECK(cudaMemcpy(feat_.p, fm.data(), sizeof(FeatMeta) * F_, cudaMemcpyHostToDevice));

    bins_.alloc(static_cast<size_t>(N_) * pitch_);
    if (pitch_ != C_) CUDA_CHECK(cudaMemset(bins_.p, 0, static_cast<size_t>(N_) * pitch_));
    CUDA_CHECK(cudaMemcpy2D(bins_.p, pitch_, bins_host, C_, C_, N_, cudaMemcpyDefault));      // host or device pointer (UVA)

    // column-major copy for the partition kernels (+C*N bytes; LGBMB200_Config.reserved bit 0 disables it)
    if (!(cfg_.reserved & 1)) {
      // a pageable H2D cudaMemcpy may return before its DMA has landed, and stream_ is a non-blocking stream:
      // make the matrix resident before the first kernel reads it
      CUDA_CHECK(cudaDeviceSynchronize());
      binsT_.alloc(static_cast<size_t>(N_) * C_);
      dim3 tg(static_cast<unsigned>((N_ + 31) / 32), static_cast<unsigned>((C_ + 31) / 32));
      k_transpose_bins<<<tg, 256, 0, stream_>>>(bins_.p, pitch_, N_, C_, binsT_.p);
      CUDA_CHECK(cudaGetLastError());
    } else {
      binsT_.release();
    }
    gq_.alloc(N_); gqo0_.alloc(N_); gqo1_.alloc(N_); idx0_.alloc(N_); idx1_.alloc(N_); flags_.alloc((static_cast<size_t>(N_) + 31) / 32 * 4 + 256);
    grad_stage_.alloc(N_); hess_stage_.alloc(N_);
    const_hess_ = is_constant_hessian != 0; hess_fill_valid_ = false;
    params_.quant_const_hess = const_hess_ ? 1 : 0;
    if (params_.quant) { ghq_.alloc(N_); ghqo0_.alloc(N_); ghqo1_.alloc(N_); } else { ghq_.release(); ghqo0_.release(); ghqo1_.release(); }
    part_blocks_ = num_sms_ * 2;
    if (part_blocks_ > 1024) part_blocks_ = 1024;
    block_left_.alloc(part_blocks_);
    prep_blocks_ = num_sms_ * 2;
    partials_.alloc(prep_blocks_);
    ctl_.alloc(1);
    CUDA_CHECK(cudaMemset(ctl_.p, 0, sizeof(Ctl)));      // exchange sequence numbers start at 0 on every rank
    // a re-Init starts from a single-GPU learner: drop the mappings of the previous shard shape (the CommBlock is sized
    // by num_data / num_features and is re-created by the next CommExport / CommPrepare)
    for (void* p : comm_opened_) cudaIpcCloseMemHandle(p);
    comm_opened_.clear();
    if (comm_local_) { cudaFree(comm_local_); comm_local_ = nullptr; }
    peers_ = CommPeers{};
    peers_.rank = 0; peers_.world = 1; peers_.flags_stride = 0;
    binsT_full_.release(); gmeta_.release();
    feature_used_.alloc(F_);
    have_feature_mask_ = false;
    bag_count_ = -1;
    CUDA_CHECK(cudaFuncSetAttribute(k_hist_a<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AShape<true>::kSmem));
    CUDA_CHECK(cudaFuncSetAttribute(k_hist_a<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AShape<false>::kSmem));
    CUDA_CHECK(cudaFuncSetAttribute(k_hist_q, cudaFuncAttributeMaxDynamicSharedMemorySize, kQSmemBytes));
    CUDA_CHECK(cudaFuncSetAttribute(k_hist_q, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    // RouteAllRows stages up to kRouteMaxSplits records (53 248 B), past the 48 KB a launch gets without opting in
    CUDA_CHECK(cudaFuncSetAttribute(k_route_rows, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    static_cast<int>(sizeof(RouteSplit) * kRouteMaxSplits)));
    BuildTensorMap();
    inited_ = true;
    AllocTreeState();
    CUDA_CHECK(cudaDeviceSynchronize());
  }

  void SetFeatureMask(const uint8_t* mask) {
    REQUIRE(inited_, "Init first");
    const bool had = have_feature_mask_;
    if (mask == nullptr) { have_feature_mask_ = false; }
    else {
      CUDA_CHECK(cudaMemcpyAsync(feature_used_.p, mask, F_, cudaMemcpyHostToDevice, stream_));
      CUDA_CHECK(cudaStreamSynchronize(stream_));
      have_feature_mask_ = true;
    }
    // the mask buffer is stable: a new mask is just new bytes; the captured graph only changes when the scan switches
    // between "no mask" and "mask"
    if (had != have_feature_mask_) InvalidateGraph();
  }

  // TreeLearner::ResetIsConstantHessian (tree_learner.h:49): GBDT::ResetTrainingData may swap the objective
  void SetConstantHessian(int is_constant_hessian) {
    REQUIRE(inited_, "Init first");
    const bool v = is_constant_hessian != 0;
    if (v == const_hess_) return;
    const_hess_ = v; hess_fill_valid_ = false;
    params_.quant_const_hess = const_hess_ ? 1 : 0;
    AllocTreeState();          // the flush scratch is sized for the histogram kernel in use; also drops the graph
  }

  void SetBagging(const int32_t* idx, int32_t n, int on_device) {
    REQUIRE(inited_, "Init first");
    if (idx == nullptr) { if (bag_count_ >= 0) InvalidateGraph(); bag_count_ = -1; return; }
    REQUIRE(n > 0 && n <= N_, "bad bagging count");
    // the bag buffer and its device-side count have stable addresses: a new bag (any size) replays the captured graph;
    // only the switch between "no bag" and "bag" changes the launch sequence
    if (bag_.n < static_cast<size_t>(N_)) { bag_.alloc(N_); bag_n_dev_.alloc(1); InvalidateGraph(); }
    CUDA_CHECK(cudaMemcpyAsync(bag_.p, idx, sizeof(int32_t) * n, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream_));
    CUDA_CHECK(cudaMemcpyAsync(bag_n_dev_.p, &n, sizeof(int32_t), cudaMemcpyHostToDevice, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    if (bag_count_ < 0) InvalidateGraph();
    bag_count_ = n;
  }

  // GOSSStrategy::Bagging on the device (goss_kernel.cuh): gradients / hessians are device arrays, modified in place;
  // the kept rows become this learner's bagging set without touching the host.
  int32_t GossSample(float* grad, float* hess, double top_rate, double other_rate, int32_t seed, int32_t iteration) {
    REQUIRE(inited_, "Init first");
    REQUIRE(top_rate > 0.0 && other_rate > 0.0 && top_rate + other_rate <= 1.0, "GOSS needs top_rate > 0, other_rate > 0, top_rate + other_rate <= 1");
    if (bag_.n < static_cast<size_t>(N_)) { bag_.alloc(N_); bag_n_dev_.alloc(1); InvalidateGraph(); }
    if (goss_state_.n == 0) { goss_state_.alloc(1); goss_hist_.alloc(256); goss_blocks_.alloc(part_blocks_); }
    GossArgs ga;
    ga.grad = grad; ga.hess = hess; ga.n = N_; ga.hist = goss_hist_.p; ga.st = goss_state_.p;
    ga.flag_words = reinterpret_cast<uint32_t*>(flags_.p); ga.block_cnt = goss_blocks_.p; ga.bag = bag_.p; ga.bag_count = bag_n_dev_.p;
    ga.top_rate = top_rate; ga.other_rate = other_rate; ga.seed = static_cast<uint32_t>(seed); ga.iter = static_cast<uint32_t>(iteration);
    k_goss_begin<<<1, 32, 0, stream_>>>(ga);
    for (int shift = 24; shift >= 0; shift -= 8) {
      k_goss_hist<<<num_sms_ * 4, kGossThreads, 0, stream_>>>(ga, shift);
      k_goss_pick<<<1, 32, 0, stream_>>>(ga, shift);
    }
    k_goss_mark<<<part_blocks_, kGossThreads, 0, stream_>>>(ga);
    k_goss_scatter<<<part_blocks_, kGossThreads, 0, stream_>>>(ga);
    launches_ += 11;
    CUDA_CHECK(cudaGetLastError());
    int32_t n = 0;
    CUDA_CHECK(cudaMemcpyAsync(&n, bag_n_dev_.p, sizeof(int32_t), cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    REQUIRE(n > 0 && n <= N_, "GOSS kept no row");
    if (bag_count_ < 0) InvalidateGraph();
    bag_count_ = n;
    return n;
  }
  void GetBag(int32_t* out, int32_t n) {
    REQUIRE(bag_count_ >= 0 && n == bag_count_, "no bagging set of that size");
    CUDA_CHECK(cudaMemcpy(out, bag_.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
  }

  void Train(const float* grad, const float* hess, int on_device, LGBMB200_Tree* out) {
    REQUIRE(inited_, "Init first");
    REQUIRE(out && out->splits && out->leaf_value && out->leaf_weight && out->leaf_count && out->leaf_depth, "null output buffers");
    const float* g = grad; const float* h = hess;
    if (!on_device) {
      CUDA_CHECK(cudaMemcpyAsync(grad_stage_.p, grad, sizeof(float) * N_, cudaMemcpyHostToDevice, stream_));
      if (const_hess_) {
        // Init(..., is_constant_hessian = true): every hessian equals hessians[0] (the reference reads only that
        // element too, dataset.cpp:1430-1437) => 4 B/row cross PCIe, not 8
        const float h0 = hess[0];
        if (!hess_fill_valid_ || h0 != hess_fill_) {
          k_fill_f32<<<num_sms_ * 4, 256, 0, stream_>>>(hess_stage_.p, h0, N_);
          ++launches_;
          CUDA_CHECK(cudaGetLastError());
          hess_fill_ = h0; hess_fill_valid_ = true;
        }
      } else {
        CUDA_CHECK(cudaMemcpyAsync(hess_stage_.p, hess, sizeof(float) * N_, cudaMemcpyHostToDevice, stream_));
      }
      g = grad_stage_.p; h = hess_stage_.p;
    }
    const int NL = params_.num_leaves;
    if (cfg_.use_cuda_graph && !profiling_) {
      if (graph_exec_ == nullptr || graph_g_ != g || graph_h_ != h) BuildGraph(g, h);
      CUDA_CHECK(cudaGraphLaunch(graph_exec_, stream_));
      launches_ += launches_per_tree_;
    } else {
      EnqueueTree(g, h);
    }
    CUDA_CHECK(cudaMemcpyAsync(h_splits_, splits_.p, sizeof(SplitRec) * (NL - 1), cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaMemcpyAsync(h_leaves_, leaves_.p, sizeof(Leaf) * NL, cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaMemcpyAsync(h_ctl_, ctl_.p, sizeof(Ctl), cudaMemcpyDeviceToHost, stream_));
    const bool renew = params_.quant && params_.quant_renew;
    if (renew) CUDA_CHECK(cudaMemcpyAsync(h_renew_, renew_out_.p, sizeof(double) * NL, cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));     // the one host sync per tree
    if (profiling_) CollectHistTimes();

    if (h_ctl_->error) throw CudaError{"feature-shard exchange timed out: a peer rank did not arrive (see LGBMB200_LearnerCommConnect)"};
    const int n_leaves = h_ctl_->num_leaves;
    out->num_leaves = n_leaves;
    out->root_sum_gradient = h_ctl_->root_sum_g; out->root_sum_hessian = h_ctl_->root_sum_h;
    // Tree::Split replay (tree.h:543-585): leaf values/weights/counts/depths, starting from the root as leaf 0
    out->leaf_value[0] = h_leaves_[0].output; out->leaf_weight[0] = h_ctl_->root_sum_h; out->leaf_count[0] = h_ctl_->root_count;
    out->leaf_depth[0] = 0;
    for (int i = 0; i < n_leaves - 1; ++i) {
      const SplitRec& r = h_splits_[i];
      LGBMB200_Split& s = out->splits[i];
      s.leaf = r.leaf; s.feature = r.feature + ((peers_.world > 1 && peers_.mode != 1) ? feature_offsets_[r.owner] : 0); s.threshold = r.threshold; s.default_left = r.default_left;
      s.left_count = r.left_count; s.right_count = r.right_count; s.gain = r.gain;
      s.left_sum_gradient = r.lsg; s.left_sum_hessian = r.lsh; s.left_output = r.lout;
      s.right_sum_gradient = r.rsg; s.right_sum_hessian = r.rsh; s.right_output = r.rout;
      const int right = i + 1;
      out->leaf_value[r.leaf] = std::isnan(r.lout) ? 0.0 : r.lout;
      out->leaf_weight[r.leaf] = r.lsh; out->leaf_count[r.leaf] = r.left_count;
      out->leaf_value[right] = std::isnan(r.rout) ? 0.0 : r.rout;
      out->leaf_weight[right] = r.rsh; out->leaf_count[right] = r.right_count;
      out->leaf_depth[right] = out->leaf_depth[r.leaf] + 1;
      out->leaf_depth[r.leaf] += 1;
    }
    if (renew) {
      // Tree::SetLeafOutput for every leaf (gradient_discretizer.cpp:255-257)
      for (int i = 0; i < n_leaves; ++i) out->leaf_value[i] = h_renew_[i];
    }
    if (params_.quant) { out->grad_scale = h_ctl_->q_gscale; out->hess_scale = h_ctl_->q_hscale; }
    else { out->grad_scale = 0.0; out->hess_scale = 0.0; }
    last_num_leaves_ = n_leaves;
  }

  void AddPredictionToScore(const double* leaf_value, int num_leaves, double* score, int on_device) {
    REQUIRE(inited_ && last_num_leaves_ > 0, "Train first");
    REQUIRE(num_leaves == last_num_leaves_, "num_leaves does not match the last trained tree");
    if (on_device) {
      CUDA_CHECK(cudaMemcpyAsync(leaf_value_dev_.p, leaf_value, sizeof(double) * num_leaves, cudaMemcpyHostToDevice, stream_));
      ScoreArgs sa{leaves_.p, idx0_.p, idx1_.p, leaf_value_dev_.p, score};
      dim3 grid(std::max(1, std::min(num_sms_ * 4, (N_ + 255) / 256)), num_leaves);
      k_add_score<<<grid, 256, 0, stream_>>>(sa);
      ++launches_;
      CUDA_CHECK(cudaGetLastError());
      CUDA_CHECK(cudaStreamSynchronize(stream_));
      return;
    }
    // host score (the link-seam path, boosting_on_gpu_ == false): ship the per-row leaf ids, add on the host.
    // Up to 255 leaves the ids travel as one byte per row (0xFF = row outside the bag), else as int32.
    const bool narrow = num_leaves <= 255;
    if (narrow) FetchLeafIndex<uint8_t>(row_leaf8_, h_row_leaf8_, 0, N_, nullptr);
    else FetchLeafIndex<int32_t>(row_leaf_, h_row_leaf_, 0, N_, nullptr);
    const int32_t* rl = h_row_leaf_;
    const uint8_t* rl8 = h_row_leaf8_;
    const int hw = static_cast<int>(std::thread::hardware_concurrency());
    const int nt = std::max(1, std::min(32, hw / std::max(1, peers_.world)));
    std::vector<std::thread> th;
    const int64_t per = (static_cast<int64_t>(N_) + nt - 1) / nt;
    for (int t = 0; t < nt; ++t) {
      th.emplace_back([=]() {
        const int64_t lo = t * per, hi = std::min<int64_t>(N_, lo + per);
        if (narrow) { for (int64_t i = lo; i < hi; ++i) { const int l = rl8[i]; if (l != 0xFF) score[i] += leaf_value[l]; } }
        else { for (int64_t i = lo; i < hi; ++i) { const int l = rl[i]; if (l >= 0) score[i] += leaf_value[l]; } }
      });
    }
    for (auto& t : th) t.join();
  }

  // every row (in the bag or not) through the last tree: score += leaf value (device score) and / or leaf ids
  void RouteAllRows(const double* leaf_value_host, int num_leaves, double* score_dev, int32_t* row_leaf_dev) {
    REQUIRE(inited_ && last_num_leaves_ > 0, "Train first");
    REQUIRE(num_leaves == last_num_leaves_, "num_leaves does not match the last trained tree");
    REQUIRE(!(peers_.world > 1 && peers_.mode != 1), "routing needs every column on this rank (single GPU or row-shard)");
    const int ns = num_leaves - 1;
    REQUIRE(ns <= kRouteMaxSplits, "too many leaves for k_route_rows");
    if (score_dev != nullptr)
      CUDA_CHECK(cudaMemcpyAsync(leaf_value_dev_.p, leaf_value_host, sizeof(double) * num_leaves, cudaMemcpyHostToDevice, stream_));
    k_route_rows<<<num_sms_ * 8, 256, sizeof(RouteSplit) * std::max(ns, 1), stream_>>>(bins_.p, pitch_, N_, splits_.p, feat_.p, ns,
                                                                                       leaf_value_dev_.p, score_dev, row_leaf_dev);
    ++launches_;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(stream_));
  }

  // leaf id of every row of the last tree into `dev` (uint8_t up to 255 leaves, else int32_t; all bits set = outside the
  // bag), then rows [lo, hi) to `out` (nullptr: to the same rows of the pinned host mirror `pinned`)
  template <typename T>
  void FetchLeafIndex(DevBuf<T>& dev, T*& pinned, int32_t lo, int32_t hi, T* out) {
    REQUIRE(inited_ && last_num_leaves_ > 0 && (sizeof(T) > 1 || last_num_leaves_ <= 255), "Train first (<= 255 leaves for 8-bit ids)");
    REQUIRE(lo >= 0 && lo <= hi && hi <= N_, "bad row range");
    if (dev.n < static_cast<size_t>(N_)) {
      dev.alloc(N_);
      if (pinned) cudaFreeHost(pinned);
      CUDA_CHECK(cudaMallocHost(&pinned, sizeof(T) * N_));
    }
    if (bag_count_ >= 0) CUDA_CHECK(cudaMemsetAsync(dev.p, 0xFF, sizeof(T) * N_, stream_));
    dim3 grid(std::max(1, std::min(num_sms_ * 4, (N_ + 255) / 256)), last_num_leaves_);
    k_leaf_index<T><<<grid, 256, 0, stream_>>>(leaves_.p, idx0_.p, idx1_.p, dev.p);
    ++launches_;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out ? out : pinned + lo, dev.p + lo, sizeof(T) * (hi - lo), cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
  }

  // leaf ids (one byte per row, 0xFF = outside the bag) of rows [lo, hi) only: N > 1 ranks that each keep a row slice of
  // the host score fetch their slice instead of all N bytes
  void GetLeafIndexRange8(int32_t lo, int32_t hi, uint8_t* out_host) { FetchLeafIndex(row_leaf8_, h_row_leaf8_, lo, hi, out_host); }
  void GetLeafIndex(int32_t* out) {
    FetchLeafIndex<int32_t>(row_leaf_, h_row_leaf_, 0, N_, nullptr);
    std::memcpy(out, h_row_leaf_, sizeof(int32_t) * N_);
  }

  void TimerStart() {
    if (!t0_) { CUDA_CHECK(cudaEventCreate(&t0_)); CUDA_CHECK(cudaEventCreate(&t1_)); }
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    CUDA_CHECK(cudaEventRecord(t0_, stream_));
  }
  float TimerStop() {
    REQUIRE(t0_ != nullptr, "TimerStart first");
    CUDA_CHECK(cudaEventRecord(t1_, stream_));
    CUDA_CHECK(cudaEventSynchronize(t1_));
    float ms = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, t0_, t1_));
    return ms;
  }

  void GetPartition(int32_t* leaf_begin, int32_t* leaf_count, int32_t* indices) {
    REQUIRE(inited_ && last_num_leaves_ > 0, "Train first");
    std::vector<int32_t> b0(N_), b1(N_);
    CUDA_CHECK(cudaMemcpy(b0.data(), idx0_.p, sizeof(int32_t) * N_, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(b1.data(), idx1_.p, sizeof(int32_t) * N_, cudaMemcpyDeviceToHost));
    for (int l = 0; l < last_num_leaves_; ++l) {
      const Leaf& L = h_leaves_[l];
      leaf_begin[l] = L.begin; leaf_count[l] = L.lcount;      // rows of the leaf held by this rank
      const std::vector<int32_t>& src = L.buf ? b1 : b0;
      std::memcpy(indices + L.begin, src.data() + L.begin, sizeof(int32_t) * L.lcount);
    }
  }

  void GetLeafHistogram(int leaf, double* out) {
    REQUIRE(inited_ && last_num_leaves_ > 0 && leaf >= 0 && leaf < last_num_leaves_, "bad leaf");
    ReadSlot(h_leaves_[leaf].slot, h_ctl_->g_inv, h_ctl_->h_inv, out);
  }

  void ConstructHistogram(const float* grad, const float* hess, int on_device, const int32_t* idx_host, int n_idx,
                          double* out, float* elapsed_ms) {
    REQUIRE(inited_, "Init first");
    const float* g = grad; const float* h = hess;
    if (!on_device) {
      CUDA_CHECK(cudaMemcpyAsync(grad_stage_.p, grad, sizeof(float) * N_, cudaMemcpyHostToDevice, stream_));
      CUDA_CHECK(cudaMemcpyAsync(hess_stage_.p, hess, sizeof(float) * N_, cudaMemcpyHostToDevice, stream_));
      hess_fill_valid_ = false;
      g = grad_stage_.p; h = hess_stage_.p;
    }
    // prep with "no bagging" semantics over all rows: packs gh and sets the fixed-point scales
    PrepArgs pa = MakePrepArgs(g, h);
    pa.bag = nullptr; pa.bag_count = nullptr;
    pa.peers.world = 1;            // stand-alone hook: local histogram only, no exchange
    k_prep<<<prep_blocks_, kPrepThreads, 0, stream_>>>(pa);
    k_root_init<<<1, 32, 0, stream_>>>(pa);
    k_quant_rows<<<prep_blocks_, kPrepThreads, 0, stream_>>>(pa);
    const int32_t* didx = nullptr;
    int n = N_;
    if (idx_host != nullptr) {
      REQUIRE(n_idx >= 0 && n_idx <= N_, "bad index count");
      CUDA_CHECK(cudaMemcpyAsync(idx1_.p, idx_host, sizeof(int32_t) * n_idx, cudaMemcpyHostToDevice, stream_));
      didx = idx1_.p; n = n_idx;
    }
    CUDA_CHECK(cudaMemsetAsync(pool_.p, 0, sizeof(long long) * slot_stride_, stream_));
    CUDA_CHECK(cudaMemsetAsync(blk_count_.p, 0, sizeof(int32_t) * hist_sets_, stream_));
    HistAArgs ha = MakeHistArgs();
    ha.explicit_n = n; ha.explicit_slot = 0; ha.explicit_idx = didx;
    cudaEvent_t e0, e1;
    CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
    CUDA_CHECK(cudaEventRecord(e0, stream_));
    LaunchHist(ha, HistQArgs{});
    CUDA_CHECK(cudaEventRecord(e1, stream_));
    launches_ += 4;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(h_ctl_, ctl_.p, sizeof(Ctl), cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    float ms = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (elapsed_ms) *elapsed_ms = ms;
    if (out) ReadSlot(0, h_ctl_->g_inv, h_ctl_->h_inv, out);
    last_num_leaves_ = 0;
  }

  // ---- feature-shard bootstrap: export this rank's CommBlock, then map every peer's
  void CommExport(uint8_t* handle_out) {
    CommPrepare();
    cudaIpcMemHandle_t hnd;
    CUDA_CHECK(cudaIpcGetMemHandle(&hnd, comm_local_));
    static_assert(sizeof(hnd) == 64, "cudaIpcMemHandle_t is 64 bytes");
    std::memcpy(handle_out, &hnd, 64);
  }
  // this rank's CommBlock (allocated on first use): what peers map (CUDA IPC between processes, plain peer access
  // between learners of one process)
  void* CommPrepare() {
    REQUIRE(inited_, "Init first");
    const int64_t stride = ((static_cast<int64_t>(N_) + 31) / 32 * 4 + 255) / 256 * 256;
    const size_t bytes = sizeof(CommBlock) + 2 * static_cast<size_t>(stride) + sizeof(FeatMeta) * static_cast<size_t>(F_);
    if (!comm_local_) {
      CUDA_CHECK(cudaMalloc(&comm_local_, bytes));
      CUDA_CHECK(cudaMemset(comm_local_, 0, bytes));
    }
    comm_stride_ = stride;
    // shard shape + layout contract behind the flag words: what a peer needs to replicate my partition columns
    {
      CommBlock* cb = reinterpret_cast<CommBlock*>(comm_local_);
      const int32_t shape[2] = {F_, C_};
      CUDA_CHECK(cudaMemcpy(&cb->num_features, shape, sizeof(shape), cudaMemcpyHostToDevice));
      CUDA_CHECK(cudaMemcpy(comm_meta_tail(cb, stride), feat_.p, sizeof(FeatMeta) * F_, cudaMemcpyDeviceToDevice));
      CUDA_CHECK(cudaDeviceSynchronize());
    }
    return comm_local_;
  }
  void CommConnect(int rank, int world, const uint8_t* handles, const int32_t* feature_offsets) {
    REQUIRE(comm_local_ != nullptr, "CommExport first");
    REQUIRE(world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world, "bad rank/world");
    void* blocks[kMaxRanks] = {nullptr};
    for (int r = 0; r < world; ++r) {
      if (r == rank) { blocks[r] = comm_local_; continue; }
      cudaIpcMemHandle_t hnd;
      std::memcpy(&hnd, handles + 64 * r, 64);
      void* p = nullptr;
      CUDA_CHECK(cudaIpcOpenMemHandle(&p, hnd, cudaIpcMemLazyEnablePeerAccess));
      blocks[r] = p;
      comm_opened_.push_back(p);
    }
    CommConnectPtrs(rank, world, blocks, feature_offsets);
  }
  // blocks[r] = rank r's CommBlock, reachable from this device (IPC mapping or peer access)
  void CommConnectPtrs(int rank, int world, void* const* blocks, const int32_t* feature_offsets) {
    REQUIRE(comm_local_ != nullptr, "CommPrepare first");
    REQUIRE(world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world, "bad rank/world");
    peers_ = CommPeers{};
    peers_.rank = rank; peers_.world = world; peers_.flags_stride = comm_stride_;
    for (int r = 0; r < world; ++r) peers_.block[r] = reinterpret_cast<CommBlock*>(r == rank ? comm_local_ : blocks[r]);
    feature_offsets_.assign(feature_offsets, feature_offsets + world + 1);
    InvalidateGraph();
  }
  const uint8_t* ColumnsPtr() const { return binsT_.p; }
  int device() const { return device_; }
  int inited_device() const { return inited_ ? device_ : (cfg_.gpu_device_id >= 0 ? cfg_.gpu_device_id : -1); }

  // feature-shard, optional: replicate every rank's column-major partition columns on every rank
  // (C_total x N bytes of HBM per GPU), so that each rank computes the go-left flags of EVERY split itself and the
  // per-split flag push + wait over NVLink disappears.  Export first, all-gather the handles, then share; the caller
  // must barrier after CommShareColumns (peers copy out of this rank's buffer).
  void CommExportColumns(uint8_t* handle_out) {
    REQUIRE(inited_ && binsT_.p != nullptr, "Init (with the column-major copy enabled) first");
    cudaIpcMemHandle_t hnd;
    CUDA_CHECK(cudaIpcGetMemHandle(&hnd, binsT_.p));
    std::memcpy(handle_out, &hnd, 64);
  }
  void CommShareColumns(const uint8_t* column_handles) {
    REQUIRE(peers_.world > 1 && peers_.mode != 1, "CommConnect (feature-shard) first");
    const int W = peers_.world;
    const uint8_t* cols[kMaxRanks] = {nullptr};
    std::vector<void*> opened;
    for (int r = 0; r < W; ++r) {
      if (r == peers_.rank) continue;
      cudaIpcMemHandle_t hnd;
      std::memcpy(&hnd, column_handles + 64 * r, 64);
      void* p = nullptr;
      CUDA_CHECK(cudaIpcOpenMemHandle(&p, hnd, cudaIpcMemLazyEnablePeerAccess));
      opened.push_back(p);
      cols[r] = static_cast<const uint8_t*>(p);
    }
    CommShareColumnsPtrs(cols);
    for (void* p : opened) cudaIpcCloseMemHandle(p);
  }
  // cols[r] = rank r's column-major copy (own entry ignored), reachable from this device
  void CommShareColumnsPtrs(const uint8_t* const* cols) {
    REQUIRE(peers_.world > 1 && peers_.mode != 1, "CommConnect (feature-shard) first");
    REQUIRE(binsT_.p != nullptr, "the column-major copy is disabled (LGBMB200_Config.reserved bit 0)");
    CUDA_CHECK(cudaStreamSynchronize(stream_));        // my own transpose has finished
    const int W = peers_.world;
    std::vector<int32_t> nf(W), nc(W), col_off(W + 1, 0), f_off(W + 1, 0);
    for (int r = 0; r < W; ++r) {
      int32_t shape[2];
      CUDA_CHECK(cudaMemcpy(shape, &peers_.block[r]->num_features, sizeof(shape), cudaMemcpyDefault));
      nf[r] = shape[0]; nc[r] = shape[1];
      REQUIRE(nf[r] >= 0 && nc[r] >= 1, "peer CommBlock carries no shard shape (CommExport on every rank first)");
      col_off[r + 1] = col_off[r] + nc[r]; f_off[r + 1] = f_off[r] + nf[r];
    }
    REQUIRE(nf[peers_.rank] == F_ && nc[peers_.rank] == C_, "own shard shape mismatch");
    binsT_full_.alloc(static_cast<size_t>(col_off[W]) * N_);
    std::vector<FeatMeta> gm(static_cast<size_t>(std::max(f_off[W], 1)));
    for (int r = 0; r < W; ++r) {
      const uint8_t* src = (r == peers_.rank) ? binsT_.p : cols[r];
      CUDA_CHECK(cudaMemcpyAsync(binsT_full_.p + static_cast<size_t>(col_off[r]) * N_, src, static_cast<size_t>(nc[r]) * N_,
                                 cudaMemcpyDefault, stream_));
      if (nf[r] > 0)
        CUDA_CHECK(cudaMemcpy(gm.data() + f_off[r], comm_meta_tail(peers_.block[r], comm_stride_), sizeof(FeatMeta) * nf[r], cudaMemcpyDefault));
      for (int f = 0; f < nf[r]; ++f) gm[f_off[r] + f].col += col_off[r];
    }
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    gmeta_.alloc(gm.size());
    CUDA_CHECK(cudaMemcpy(gmeta_.p, gm.data(), sizeof(FeatMeta) * gm.size(), cudaMemcpyHostToDevice));
    peers_.mode = 2;
    peers_.gmeta = gmeta_.p;
    for (int r = 0; r < W; ++r) peers_.feat_off[r] = f_off[r];
    InvalidateGraph();
  }

  // row-shard bootstrap: additionally export the histogram pool, whose peer copies k_scan sums over NVLink
  void CommExportPool(uint8_t* handle_out) {
    REQUIRE(inited_, "Init first");
    cudaIpcMemHandle_t hnd;
    CUDA_CHECK(cudaIpcGetMemHandle(&hnd, pool_.p));
    std::memcpy(handle_out, &hnd, 64);
  }
  void CommConnectRows(int rank, int world, const uint8_t* comm_handles, const uint8_t* pool_handles) {
    const std::vector<int32_t> dummy(world + 1, 0);
    CommConnect(rank, world, comm_handles, dummy.data());
    peers_.mode = 1;
    // feature slice reduced + scanned by this rank: contiguous, balanced by count
    const int base = F_ / world, extra = F_ % world;
    peers_.f_lo = rank * base + std::min(rank, extra);
    peers_.f_cnt = base + (rank < extra ? 1 : 0);
    for (int r = 0; r < world; ++r) {
      if (r == rank) { peers_.pool[r] = pool_.p; continue; }
      cudaIpcMemHandle_t hnd;
      std::memcpy(&hnd, pool_handles + 64 * r, 64);
      void* p = nullptr;
      CUDA_CHECK(cudaIpcOpenMemHandle(&p, hnd, cudaIpcMemLazyEnablePeerAccess));
      peers_.pool[r] = reinterpret_cast<long long*>(p);
      comm_opened_.push_back(p);
    }
    InvalidateGraph();
  }

  void L2Gradients(const double* score, const float* label, float* grad, float* hess, int n) {
    k_l2_gradients<<<num_sms_ * 4, 256, 0, stream_>>>(score, label, grad, hess, n);
    ++launches_;
    CUDA_CHECK(cudaGetLastError());
  }

  void BinaryGradients(const double* score, const float* label, float* grad, float* hess, int n, double sigmoid) {
    k_binary_gradients<<<num_sms_ * 4, 256, 0, stream_>>>(score, label, grad, hess, n, sigmoid);
    ++launches_;
    CUDA_CHECK(cudaGetLastError());
  }

  void SetProfiling(int enable) {
    profiling_ = enable != 0;
    if (profiling_ && hist_events_.empty()) {
      hist_events_.resize(8 * static_cast<size_t>(params_.num_leaves) + 8);
      prof_kind_.assign(hist_events_.size(), 0);
      for (auto& e : hist_events_) CUDA_CHECK(cudaEventCreate(&e));
    }
  }
  void HistStats(int reset, double* ms, double* rows, int64_t* launches) {
    if (ms) *ms = hist_ms_;
    if (rows) *rows = hist_rows_;
    if (launches) *launches = hist_launches_;
    if (reset) { hist_ms_ = 0; hist_rows_ = 0; hist_launches_ = 0; for (double& v : prof_ms_) v = 0; }
  }
  void ProfileByKind(double* out9) { for (int i = 0; i < kProfKinds; ++i) out9[i] = prof_ms_[i]; }
  int64_t launches() const { return launches_; }
  cudaStream_t stream() const { return stream_; }

 private:
  void AllocTreeState() {
    const int NL = params_.num_leaves;
    slot_stride_ = static_cast<int64_t>(Cpad_) * kBinsPerColumn * 2;
    pool_.alloc(static_cast<size_t>(slot_stride_) * NL);
    leaves_.alloc(NL); splits_.alloc(NL); cand_.alloc(2 * static_cast<size_t>(F_));
    splittable_.alloc(static_cast<size_t>(NL) * F_);
    splittable_new_.alloc(2 * static_cast<size_t>(F_));
    block_best_.alloc(2 * static_cast<size_t>((F_ + kScanWarps - 1) / kScanWarps));
    leaf_value_dev_.alloc(NL);
    // flush scratch of k_hist_a: per column-group set, one block per (CTA, flush interval) — see HistAArgs
    {
      const int G = ConstHessHist() ? AShape<true>::G : AShape<false>::G;
      const size_t blk = ConstHessHist() ? AShape<true>::kTables : AShape<false>::kTables;
      hist_sets_ = Cpad_ / kColGroup / G;
      blk_cap_ = (N_ / kARows) / (kAFlushRows / kARows) + num_sms_ + 2;
      scratch_.alloc(static_cast<size_t>(hist_sets_) * blk_cap_ * blk);
      blk_count_.alloc(static_cast<size_t>(NL) * hist_sets_);
    }
    renew_partial_.alloc(static_cast<size_t>(NL) * kRenewBlocks * 2); renew_out_.alloc(NL);
    if (h_renew_) cudaFreeHost(h_renew_);
    CUDA_CHECK(cudaMallocHost(&h_renew_, sizeof(double) * NL));
    if (h_splits_) { cudaFreeHost(h_splits_); cudaFreeHost(h_leaves_); cudaFreeHost(h_ctl_); }
    CUDA_CHECK(cudaMallocHost(&h_splits_, sizeof(SplitRec) * NL));
    CUDA_CHECK(cudaMallocHost(&h_leaves_, sizeof(Leaf) * NL));
    CUDA_CHECK(cudaMallocHost(&h_ctl_, sizeof(Ctl)));
    for (auto& e : hist_events_) cudaEventDestroy(e);
    hist_events_.clear();
    if (profiling_) SetProfiling(1);
    InvalidateGraph();
  }

  PrepArgs MakePrepArgs(const float* g, const float* h) {
    PrepArgs pa;
    pa.grad = g; pa.hess = h; pa.gq = gq_.p; pa.idx0 = idx0_.p;
    pa.bag = bag_count_ >= 0 ? bag_.p : nullptr; pa.bag_count = bag_count_ >= 0 ? bag_n_dev_.p : nullptr;
    pa.num_data = N_; pa.partials = partials_.p; pa.leaves = leaves_.p; pa.ctl = ctl_.p; pa.params = params_;
    pa.max_leaves = params_.num_leaves; pa.num_partials = prep_blocks_; pa.peers = peers_;
    pa.ghq = PackedQuantHist() ? ghq_.p : nullptr;
    return pa;
  }
  HistAArgs MakeHistArgs() {
    HistAArgs ha;
    ha.bins = bins_.p; ha.pitch = pitch_; ha.gq = gq_.p; ha.gqo0 = nullptr; ha.gqo1 = nullptr;      // gqo*: set by EnqueueTree
    ha.idx0 = idx0_.p; ha.idx1 = idx1_.p;
    ha.leaves = leaves_.p; ha.ctl = ctl_.p; ha.pool = reinterpret_cast<unsigned long long*>(pool_.p);
    ha.slot_stride = slot_stride_; ha.num_colgroups = Cpad_ / kColGroup;
    ha.scratch = scratch_.p; ha.blk_count = blk_count_.p; ha.blk_cap = blk_cap_;
    static const float split_k = std::getenv("LGBMB200_SPLIT_K") ? static_cast<float>(std::atof(std::getenv("LGBMB200_SPLIT_K"))) : 0.044f;
    ha.split_k = split_k;
    ha.explicit_n = -1; ha.explicit_slot = 0; ha.explicit_idx = nullptr;
    ha.use_tma = have_tmap_ ? 1 : 0;
    // L2 prefetch distance of the gathered passes, in stages of one producer warp (LGBMB200_PF overrides it)
    static const int pf_stages = std::getenv("LGBMB200_PF") ? std::atoi(std::getenv("LGBMB200_PF")) : 4;
    ha.l2_prefetch = pf_stages;
    return ha;
  }
  // the packed-cell kernel of quantized training keeps the round-1 work mapping (hist_common.cuh)
  HistQArgs MakeHistQArgs() {
    HistQArgs qa;
    HistArgs& ha = qa.h;
    ha.bins = bins_.p; ha.pitch = pitch_; ha.idx0 = idx0_.p; ha.idx1 = idx1_.p;
    ha.leaves = leaves_.p; ha.ctl = ctl_.p; ha.pool = reinterpret_cast<unsigned long long*>(pool_.p);
    ha.slot_stride = slot_stride_; ha.num_colgroups = Cpad_ / kColGroup; ha.min_rows_per_item = 64;
    ha.explicit_n = -1; ha.explicit_slot = 0; ha.explicit_idx = nullptr;
    ha.use_tma = have_tmap_ ? 1 : 0;
    ha.map_mode = 1;
    ha.l2_prefetch = 8;
    ha.ghqo0 = nullptr; ha.ghqo1 = nullptr;
    qa.ghq = ghq_.p;
    qa.flush_rows = ((65535 / std::max(1, params_.quant_bins)) / kStageRows) * kStageRows;
    return qa;
  }

  // 2-D tensor map over the row-major bin matrix {Cpad, N} with a {32 columns, 32 rows} box, for the TMA tile
  // loads of contiguous (root) stages.  cuTensorMapEncodeTiled is fetched from the driver at run time, so the
  // library keeps depending on libcudart only.  LGBMB200_DEBUG bit 2 turns TMA staging off.
  void BuildTensorMap() {
    have_tmap_ = false;
    std::memset(&tmap_, 0, sizeof(tmap_));
    if (DebugBits() & 2) return;
    typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || fn == nullptr ||
        qres != cudaDriverEntryPointSuccess) { cudaGetLastError(); return; }
    const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(Cpad_), static_cast<cuuint64_t>(N_)};
    const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(pitch_)};
    const cuuint32_t box[2] = {kColGroup, kStageRows};
    const cuuint32_t estride[2] = {1, 1};
    const CUresult r = reinterpret_cast<EncodeTiled>(fn)(&tmap_, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, bins_.p, gdim, gstride, box, estride,
                                                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                         CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    have_tmap_ = (r == CUDA_SUCCESS);
    // the constant-hessian histogram kernel stages two column groups per row: box = {64 columns, 32 rows}
    std::memset(&tmap2_, 0, sizeof(tmap2_));
    if (have_tmap_) {
      const cuuint32_t box2[2] = {2 * kColGroup, kStageRows};
      const CUresult r2 = reinterpret_cast<EncodeTiled>(fn)(&tmap2_, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, bins_.p, gdim, gstride, box2, estride,
                                                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                            CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      have_tmap_ = (r2 == CUDA_SUCCESS);
    }
  }

  // quantized training: packed 16:16 cells whenever a flush interval of at least 4096 rows keeps both fields in
  // range (num_grad_quant_bins <= 15; LGBMB200_DEBUG bit 64 forces the general kernel for A/B runs)
  bool PackedQuantHist() const { return params_.quant && params_.quant_bins <= 15 && !(DebugBits() & 64); }
  // constant hessian (Init's flag): the count-and-scale kernel; quantized training discretizes the hessian to 1 then too,
  // but keeps the general kernel (its pool holds raw integer sums)
  bool ConstHessHist() const { return const_hess_ && !params_.quant; }

  // histogram of the current smaller leaf: accumulate (k_hist_a dumps raw table blocks) + reduce into the pool slot;
  // the packed-cell kernel of quantized training still adds into a zeroed slot with RED.ADD.64
  void LaunchHist(const HistAArgs& ha, const HistQArgs& qa) {
    if (PackedQuantHist()) { k_hist_q<<<num_sms_ * 2, kHistThreads, kQSmemBytes, stream_>>>(qa, tmap_); return; }
    // k_hist_reduce: warps per 32-column row of cells such that the grid has about two CTAs per SM — one warp per row when
    // the shard is wide (C3 on one GPU: 4096 rows), all eight when a GPU holds two sets (its share of C3 at 8 GPUs)
    auto reduce_grid = [&](int rows_total, int* wpr) {
      int w = 1;
      while (w < kReduceWarps && rows_total * w / kReduceWarps < 2 * num_sms_) w *= 2;
      *wpr = w;
      return dim3(static_cast<unsigned>((rows_total * w + kReduceWarps - 1) / kReduceWarps));
    };
    int wpr = 1;
    if (ConstHessHist()) {
      k_hist_a<true><<<num_sms_, kAThreads, AShape<true>::kSmem, stream_>>>(ha, tmap2_);
      const dim3 g = reduce_grid(hist_sets_ * AShape<true>::G * 128, &wpr);
      k_hist_reduce<true><<<g, kReduceWarps * 32, 0, stream_>>>(ha, wpr);
    } else {
      k_hist_a<false><<<num_sms_, kAThreads, AShape<false>::kSmem, stream_>>>(ha, tmap_);
      const dim3 g = reduce_grid(hist_sets_ * kBinsPerColumn, &wpr);
      k_hist_reduce<false><<<g, kReduceWarps * 32, 0, stream_>>>(ha, wpr);
    }
    ++launches_;
  }

  // The fixed per-tree launch sequence (see file header).
  void EnqueueTree(const float* g, const float* h) {
    const int NL = params_.num_leaves;
    PrepArgs pa = MakePrepArgs(g, h);
    HistAArgs ha = MakeHistArgs();
    HistQArgs qa = MakeHistQArgs();
    ScanArgs sa;
    sa.feat = feat_.p; sa.feature_used = have_feature_mask_ ? feature_used_.p : nullptr; sa.num_features = F_;
    sa.params = params_; sa.leaves = leaves_.p; sa.ctl = ctl_.p; sa.pool = pool_.p; sa.slot_stride = slot_stride_;
    sa.splittable = splittable_.p; sa.splittable_new = splittable_new_.p; sa.cand = cand_.p; sa.block_best = block_best_.p;
    sa.peers = peers_;
    const bool row_mode = peers_.world > 1 && peers_.mode == 1;
    const int scan_blocks = ((row_mode ? peers_.f_cnt : F_) + kScanWarps - 1) / kScanWarps;
    SelectArgs se{feat_.p, F_, NL, leaves_.p, ctl_.p, cand_.p, block_best_.p, scan_blocks, splittable_.p, splittable_new_.p, peers_};
    PartArgs pt;
    pt.bins = bins_.p; pt.binsT = peers_.mode == 2 ? binsT_full_.p : binsT_.p; pt.num_data = N_; pt.pitch = pitch_; pt.idx0 = idx0_.p; pt.idx1 = idx1_.p; pt.flag_words = reinterpret_cast<uint32_t*>(flags_.p);
    pt.block_left = block_left_.p; pt.leaves = leaves_.p; pt.ctl = ctl_.p; pt.splits = splits_.p; pt.params = params_;
    pt.peers = peers_;
    const bool ordered = !(DebugBits() & 256);
    const bool packed = PackedQuantHist();
    pt.gh = gq_.p; pt.gho0 = (ordered && !packed) ? gqo0_.p : nullptr; pt.gho1 = (ordered && !packed) ? gqo1_.p : nullptr;
    pt.ghq = ghq_.p; pt.ghqo0 = (ordered && packed) ? ghqo0_.p : nullptr; pt.ghqo1 = (ordered && packed) ? ghqo1_.p : nullptr;
    ha.gqo0 = pt.gho0; ha.gqo1 = pt.gho1; qa.h.ghqo0 = pt.ghqo0; qa.h.ghqo1 = pt.ghqo1;
    prof_n_ = 0;
    Stamp(kProfStart);

    const bool quant = params_.quant != 0;
    REQUIRE(!(quant && row_mode), "use_quantized_grad is not supported in row-shard mode");
    k_prep<<<prep_blocks_, kPrepThreads, 0, stream_>>>(pa);
    if (quant) {
      // GradientDiscretizer::DiscretizeGradients: scales from the maxima k_prep just reduced, then int8 (g,h)
      k_quant_scales<<<1, 32, 0, stream_>>>(pa);
      k_quantize<<<prep_blocks_, kPrepThreads, 0, stream_>>>(pa);
      launches_ += 2;
    }
    k_root_init<<<1, 32, 0, stream_>>>(pa);
    if (!quant) { k_quant_rows<<<prep_blocks_, kPrepThreads, 0, stream_>>>(pa); ++launches_; }     // per-tree fixed point of (g, h)
    CUDA_CHECK(cudaMemsetAsync(splittable_.p, 1, static_cast<size_t>(NL) * F_, stream_));
    launches_ += 2;
    Stamp(kProfPrep);
    if (PackedQuantHist()) {
      // k_hist_q adds into its slot: one memset for every histogram slot this tree can use (slot i is filled by iteration i)
      CUDA_CHECK(cudaMemsetAsync(pool_.p, 0, sizeof(long long) * slot_stride_ * static_cast<size_t>(NL - 1), stream_));
    } else {
      // k_hist_a / k_hist_reduce overwrite their slot; only the per-pass block counters start from zero
      CUDA_CHECK(cudaMemsetAsync(blk_count_.p, 0, sizeof(int32_t) * static_cast<size_t>(NL) * hist_sets_, stream_));
    }
    Stamp(kProfMemset);
    for (int it = 0; it < NL - 1 + 1; ++it) {
      // it == 0: root pass; it >= 1: apply split it-1, then find splits for its two children
      if (it > 0) {
        // (a single cooperative launch with a grid-wide barrier between the two phases was measured no faster than the
        // two launches — under graph replay a launch boundary costs no more than the barrier — and was not kept)
        k_part_flags<<<part_blocks_, kPartThreads, 0, stream_>>>(pt);
        Stamp(kProfPartFlags);
        k_part_scatter<<<part_blocks_, kPartThreads, 0, stream_>>>(pt);
        Stamp(kProfPartScatter);
        launches_ += 2;
        if (it == NL - 1) break;   // the tree is full: no need to look for further splits
      }
      LaunchHist(ha, qa);
      Stamp(kProfHist);
      if (row_mode) { k_hist_signal<<<1, 32, 0, stream_>>>(peers_, ctl_.p); ++launches_; }
      if (row_mode) k_scan<true, false><<<dim3(std::max(scan_blocks, 1), 1), kScanWarps * 32, 0, stream_>>>(sa);
      else if (quant) k_scan<false, true><<<dim3(std::max(scan_blocks, 1), 2), kScanWarps * 32, 0, stream_>>>(sa);
      else k_scan<false, false><<<dim3(std::max(scan_blocks, 1), 2), kScanWarps * 32, 0, stream_>>>(sa);
      Stamp(kProfScan);
      k_select<<<1, 256, 0, stream_>>>(se);
      Stamp(kProfSelect);
      launches_ += 3;
    }
    if (quant && params_.quant_renew) {
      // quant_train_renew_leaf: leaf outputs from the ORIGINAL gradients (g, h are still untouched: k_quantize
      // only rewrote the packed gh array)
      RenewArgs ra{g, h, leaves_.p, ctl_.p, idx0_.p, idx1_.p, renew_partial_.p, renew_out_.p, params_};
      k_renew_leaf<<<dim3(kRenewBlocks, NL), 256, 0, stream_>>>(ra);
      k_renew_leaf_finish<<<(NL + 127) / 128, 128, 0, stream_>>>(ra, kRenewBlocks);
      launches_ += 2;
    }
    CUDA_CHECK(cudaGetLastError());
  }

  void BuildGraph(const float* g, const float* h) {
    InvalidateGraph();
    const int64_t before = launches_;
    CUDA_CHECK(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
    try {
      EnqueueTree(g, h);
    } catch (...) {
      cudaGraph_t junk = nullptr;
      cudaStreamEndCapture(stream_, &junk);
      if (junk) cudaGraphDestroy(junk);
      throw;
    }
    CUDA_CHECK(cudaStreamEndCapture(stream_, &graph_));
    CUDA_CHECK(cudaGraphInstantiate(&graph_exec_, graph_, 0));
    launches_per_tree_ = launches_ - before;
    launches_ = before;
    graph_g_ = g; graph_h_ = h;
  }

  void InvalidateGraph() {
    if (graph_exec_) { cudaGraphExecDestroy(graph_exec_); graph_exec_ = nullptr; }
    if (graph_) { cudaGraphDestroy(graph_); graph_ = nullptr; }
  }

  enum ProfKind { kProfStart = 0, kProfPrep, kProfPartFlags, kProfPartCount, kProfPartScatter, kProfMemset, kProfHist, kProfScan, kProfSelect, kProfKinds };
  // profiling mode: an event after every launch; the segment since the previous event is charged to `kind`
  void Stamp(int kind) {
    if (!profiling_) return;
    if (prof_n_ >= static_cast<int>(hist_events_.size())) return;
    CUDA_CHECK(cudaEventRecord(hist_events_[prof_n_], stream_));
    prof_kind_[prof_n_] = kind;
    ++prof_n_;
  }
  void CollectHistTimes() {
    // smaller-leaf row counts of every histogram pass are recoverable from the split records
    int hist_launches = 0;
    for (int i = 1; i < prof_n_; ++i) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, hist_events_[i - 1], hist_events_[i]) != cudaSuccess) continue;
      prof_ms_[prof_kind_[i]] += ms;
      if (prof_kind_[i] == kProfHist) { hist_ms_ += ms; ++hist_launches; }
    }
    hist_events_used_ = hist_launches;
    const int n_leaves = h_ctl_->num_leaves;
    double rows = h_ctl_->root_count;
    for (int i = 0; i < n_leaves - 1; ++i) {
      if (i == params_.num_leaves - 2) break;   // children of the last split are never histogrammed
      rows += std::min(h_splits_[i].left_count, h_splits_[i].right_count);
    }
    hist_rows_ += rows;
    hist_launches_ += hist_events_used_;
  }

  void ReadSlot(int slot, double g_inv, double h_inv, double* out) {
    std::vector<long long> tmp(static_cast<size_t>(C_) * kBinsPerColumn * 2);
    CUDA_CHECK(cudaMemcpy(tmp.data(), pool_.p + static_cast<size_t>(slot) * slot_stride_, sizeof(long long) * tmp.size(), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < tmp.size(); i += 2) { out[i] = static_cast<double>(tmp[i]) * g_inv; out[i + 1] = static_cast<double>(tmp[i + 1]) * h_inv; }
  }

  void Destroy() {
    InvalidateGraph();
    for (auto& e : hist_events_) cudaEventDestroy(e);
    hist_events_.clear();
    if (h_splits_) { cudaFreeHost(h_splits_); cudaFreeHost(h_leaves_); cudaFreeHost(h_ctl_); h_splits_ = nullptr; }
    for (void* p : comm_opened_) cudaIpcCloseMemHandle(p);
    comm_opened_.clear();
    if (comm_local_) { cudaFree(comm_local_); comm_local_ = nullptr; }
    if (h_row_leaf_) { cudaFreeHost(h_row_leaf_); h_row_leaf_ = nullptr; }
    if (h_row_leaf8_) { cudaFreeHost(h_row_leaf8_); h_row_leaf8_ = nullptr; }
    if (h_renew_) { cudaFreeHost(h_renew_); h_renew_ = nullptr; }
    if (t0_) { cudaEventDestroy(t0_); cudaEventDestroy(t1_); t0_ = nullptr; }
    if (stream_) { cudaStreamDestroy(stream_); stream_ = nullptr; }
  }

  LGBMB200_Config cfg_{};
  Params params_{};
  bool inited_ = false;
  int device_ = 0, num_sms_ = 132;
  cudaStream_t stream_ = nullptr;
  int N_ = 0, C_ = 0, F_ = 0, Cpad_ = 0;
  int64_t pitch_ = 0, slot_stride_ = 0;
  int part_blocks_ = 264, prep_blocks_ = 264;
  DevBuf<FeatMeta> feat_;
  DevBuf<uint8_t> binsT_full_;     // mode 2: [sum of every rank's columns][N]
  DevBuf<FeatMeta> gmeta_;
  DevBuf<uint8_t> bins_, binsT_, flags_, feature_used_, splittable_, splittable_new_;
  DevBuf<BlockBest> block_best_;
  DevBuf<unsigned char> scratch_;       // k_hist_a flush blocks [sets][blk_cap][table image]
  DevBuf<int32_t> blk_count_;
  int hist_sets_ = 0, blk_cap_ = 0;
  DevBuf<int2> gq_, gqo0_, gqo1_;       // per-tree fixed-point (g,h) by row id; leaf-ordered copies parallel to idx0_/idx1_
  DevBuf<int32_t> ghqo0_, ghqo1_;
  static constexpr int kRenewBlocks = 64;
  DevBuf<double> renew_partial_, renew_out_;
  DevBuf<int32_t> ghq_;            // quantized training: packed (g << 16) + h per row
  double* h_renew_ = nullptr;
  DevBuf<float> grad_stage_, hess_stage_;
  bool const_hess_ = false, hess_fill_valid_ = false;
  float hess_fill_ = 0.f;
  DevBuf<double> leaf_value_dev_;
  DevBuf<int32_t> idx0_, idx1_, block_left_, bag_, bag_n_dev_, row_leaf_, goss_blocks_;
  DevBuf<GossState> goss_state_;
  DevBuf<uint32_t> goss_hist_;
  int32_t* h_row_leaf_ = nullptr;
  DevBuf<uint8_t> row_leaf8_;
  uint8_t* h_row_leaf8_ = nullptr;
  cudaEvent_t t0_ = nullptr, t1_ = nullptr;
  DevBuf<PartialSum> partials_;
  CommPeers peers_{};
  CUtensorMap tmap_;
  bool have_tmap_ = false;
  CUtensorMap tmap2_;
  void* comm_local_ = nullptr;
  int64_t comm_stride_ = 0;
  std::vector<void*> comm_opened_;
  std::vector<int32_t> feature_offsets_;
  DevBuf<Ctl> ctl_;
  DevBuf<Leaf> leaves_;
  DevBuf<SplitRec> splits_;
  DevBuf<Cand> cand_;
  DevBuf<long long> pool_;
  SplitRec* h_splits_ = nullptr;
  Leaf* h_leaves_ = nullptr;
  Ctl* h_ctl_ = nullptr;
  bool have_feature_mask_ = false;
  int bag_count_ = -1;
  int last_num_leaves_ = 0;
  cudaGraph_t graph_ = nullptr;
  cudaGraphExec_t graph_exec_ = nullptr;
  const float* graph_g_ = nullptr;
  const float* graph_h_ = nullptr;
  int64_t launches_ = 0, launches_per_tree_ = 0;
  bool profiling_ = false;
  std::vector<cudaEvent_t> hist_events_;
  int hist_events_used_ = 0;
  int prof_n_ = 0;
  std::vector<int> prof_kind_;
  double prof_ms_[16] = {0};
  double hist_ms_ = 0, hist_rows_ = 0;
  int64_t hist_launches_ = 0;
};

}  // namespace b200

// ---------------------------------------------------------------------------------------------------------------------
// Dataset construction (SURVEY.md §8 f-3): host-side mappers / bundles + the device value->bin pass, see binning.cuh
#include "binning.cuh"

namespace b200 {

// Host -> device streaming of a pageable matrix: chunks are copied by a few host threads into one of two pinned buffers
// and sent with cudaMemcpyAsync (a pageable cudaMemcpyAsync is slow and blocks the host; pinned, the link
// speed).  Filling buffer k overlaps the transfer + kernel of the chunk before it.
class PinnedStager {
 public:
  ~PinnedStager() { for (int i = 0; i < 2; ++i) { if (buf_[i]) cudaFreeHost(buf_[i]); if (ev_[i]) cudaEventDestroy(ev_[i]); } }
  void Reserve(size_t bytes) {
    if (bytes <= cap_) return;
    for (int i = 0; i < 2; ++i) {
      if (buf_[i]) cudaFreeHost(buf_[i]);
      CUDA_CHECK(cudaMallocHost(&buf_[i], bytes));
      if (!ev_[i]) CUDA_CHECK(cudaEventCreateWithFlags(&ev_[i], cudaEventDisableTiming));
    }
    cap_ = bytes;
  }
  // copy `bytes` from pageable `src` to `dst_dev` on `st` through pinned buffer `k & 1`
  void Send(int k, void* dst_dev, const void* src, size_t bytes, cudaStream_t st) {
    const int b = k & 1;
    if (used_[b]) CUDA_CHECK(cudaEventSynchronize(ev_[b]));       // the transfer that last read this buffer has finished
    const int nt = static_cast<int>(std::max<size_t>(1, std::min<size_t>(8, bytes >> 22)));
    if (nt == 1) std::memcpy(buf_[b], src, bytes);
    else {
      std::vector<std::thread> pool;
      const size_t per = (bytes / nt + 63) / 64 * 64;
      for (int t = 0; t < nt; ++t) {
        const size_t lo = std::min(bytes, per * t), hi = std::min(bytes, per * (t + 1));
        pool.emplace_back([=]() { if (hi > lo) std::memcpy(static_cast<char*>(buf_[b]) + lo, static_cast<const char*>(src) + lo, hi - lo); });
      }
      for (auto& th : pool) th.join();
    }
    CUDA_CHECK(cudaMemcpyAsync(dst_dev, buf_[b], bytes, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaEventRecord(ev_[b], st));
    used_[b] = true;
  }

 private:
  void* buf_[2] = {nullptr, nullptr};
  cudaEvent_t ev_[2] = {nullptr, nullptr};
  bool used_[2] = {false, false};
  size_t cap_ = 0;
};

class BinnerCtx {
 public:
  explicit BinnerCtx(const LGBMB200_BinConfig& c) : device_(c.gpu_device_id), binner_(ToCfg(c)) {}
  ~BinnerCtx() { for (auto& s : streams_) if (s) cudaStreamDestroy(s); }
  int device() const { return device_; }

  void Fit(const void* data, int dtype, int64_t nrow, int32_t ncol, int row_major) {
    REQUIRE(data != nullptr, "null matrix");
    REQUIRE(dtype == 0 || dtype == 1, "data_type must be 0 (float32) or 1 (float64)");
    binner_.Fit(data, dtype, nrow, ncol, row_major != 0);
    uploaded_ = false; fitted_ = true;
  }
  void GetLayout(LGBMB200_Layout* out) const {
    REQUIRE(fitted_, "Fit first");
    const BinTable& t = binner_.table();
    out->num_data = binner_.num_data(); out->num_columns = t.num_columns; out->num_features = t.num_features;
    out->feat_column = t.feat_column.data(); out->feat_lo = t.feat_lo.data(); out->feat_num_bin = t.feat_num_bin.data();
    out->feat_most_freq_bin = t.feat_mfb.data(); out->feat_default_bin = t.feat_default.data();
    out->feat_missing_type = t.feat_missing.data(); out->feat_real_index = t.feat_real.data();
  }
  void GetBounds(int f, double* upper, int32_t* num_bin) const {
    REQUIRE(fitted_, "Fit first");
    const BinTable& t = binner_.table();
    REQUIRE(f >= 0 && f < t.num_features, "bad feature index");
    const BinMapperB& m = binner_.mappers()[t.feat_real[f]];
    if (num_bin) *num_bin = m.num_bin;
    if (upper) std::memcpy(upper, m.upper.data(), sizeof(double) * m.num_bin);
  }
  int32_t GetSampleRows(int32_t* out) const {
    REQUIRE(fitted_, "Fit first");
    const std::vector<int>& r = binner_.sample_rows();
    if (out) std::memcpy(out, r.data(), sizeof(int32_t) * r.size());
    return static_cast<int32_t>(r.size());
  }

  // The N x F pass on the device.  `data` is row-major [nrow x num_total_features]; host data is streamed in row chunks
  // (copy of chunk i+1 overlaps the kernel of chunk i on the other stream); `out` is [nrow x num_columns] bytes.
  void Transform(const void* data, int dtype, int64_t nrow, int data_on_device, uint8_t* out, int out_on_device, float* elapsed_ms) {
    REQUIRE(fitted_, "Fit first");
    REQUIRE(data != nullptr && out != nullptr && nrow > 0, "bad argument");
    REQUIRE(dtype == 0 || dtype == 1, "data_type must be 0 (float32) or 1 (float64)");
    if (device_ >= 0) CUDA_CHECK(cudaSetDevice(device_));
    int dev = 0;
    CUDA_CHECK(cudaGetDevice(&dev));
    const int sms = DeviceSms(dev);
    Upload();
    const BinTable& t = binner_.table();
    const int64_t ncol = t.num_total_features, C = t.num_columns;
    const size_t esize = dtype == 0 ? 4 : 8;
    int64_t chunk = std::max<int64_t>(1024, (static_cast<int64_t>(128) << 20) / static_cast<int64_t>(ncol * esize));
    chunk = std::min(chunk, nrow);
    if (data_on_device && out_on_device) chunk = nrow;          // nothing to stage: one launch over all rows
    for (auto& s : streams_) if (!s) CUDA_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    DevBuf<unsigned char> dx[2], dout[2];
    if (!data_on_device) { for (auto& b : dx) b.alloc(static_cast<size_t>(chunk) * ncol * esize); stager_.Reserve(static_cast<size_t>(chunk) * ncol * esize); }
    if (!out_on_device) for (auto& b : dout) b.alloc(static_cast<size_t>(chunk) * C);
    const BinDevTable ro{d_ro_real_.p, d_ro_lo_.p, d_ro_num_bin_.p, d_ro_mfb_.p, d_ro_missing_.p, d_ro_bound_first_.p, d_ro_bound_count_.p,
                         d_bounds32_.p, d_bounds64_.p, static_cast<int32_t>(t.num_features)};
    // max_bin <= 255 and search_bounds_smem's depth <= 8 bound a 32-feature tile to 32 * vb_slots(8) bound words (67 KB as
    // doubles) plus about 20 KB of row tile, output tile and feature records
    const size_t smem = static_cast<size_t>(max_bounds_) * esize + sizeof(VbFeat) * max_feats_ + static_cast<size_t>(kVbRows) * (kVbCols + 1) * esize +
                        static_cast<size_t>(kVbRows) * (kVbCols / 4 + 1) * 4;
    REQUIRE(smem <= 200 * 1024, "k_value_to_bin_tile would need more than 200 KB of shared memory");
    cudaEvent_t e0, e1, ej;
    CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1)); CUDA_CHECK(cudaEventCreateWithFlags(&ej, cudaEventDisableTiming));
    CUDA_CHECK(cudaDeviceSynchronize());
    CUDA_CHECK(cudaEventRecord(e0, streams_[0]));
    CUDA_CHECK(cudaStreamWaitEvent(streams_[1], e0, 0));
    int k = 0;
    for (int64_t r0 = 0; r0 < nrow; r0 += chunk, ++k) {
      const int64_t rows = std::min(chunk, nrow - r0);
      cudaStream_t st = streams_[k & 1];
      const unsigned char* src = static_cast<const unsigned char*>(data) + static_cast<size_t>(r0) * ncol * esize;
      if (!data_on_device) {
        stager_.Send(k, dx[k & 1].p, src, static_cast<size_t>(rows) * ncol * esize, st);
        src = dx[k & 1].p;
      }
      uint8_t* dst = out_on_device ? out + r0 * C : dout[k & 1].p;
      // Step 1 reads the matrix in REAL feature order (coalesced whatever the stored column order is) and writes one byte
      // per feature; step 2 (k_bundle_columns) moves the bytes to their stored columns.  Both run over row pieces whose
      // byte image fits L2, so the intermediate never reaches DRAM.  Identity layouts skip step 2.
      const int64_t Fu = t.num_features, Fp = (Fu + 15) / 16 * 16;        // Fp: row pitch of the intermediate (16-byte rows)
      const bool direct = t.identity_order;
      // pieces of <= 16 MB of intermediate: it and the piece's stored columns stay well inside the 50 MB L2 of an H100
      const int64_t piece = direct ? rows : std::max<int64_t>(kVbRows, std::min<int64_t>(rows, (static_cast<int64_t>(16) << 20) / Fp / kVbRows * kVbRows));
      if (!direct && tmp_[k & 1].n < static_cast<size_t>(piece * Fp)) tmp_[k & 1].alloc(static_cast<size_t>(piece * Fp));
      int per_sm = 1;
      if (dtype == 0) {
        CUDA_CHECK(cudaFuncSetAttribute(k_value_to_bin_tile<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_value_to_bin_tile<float>, kVbThreads, smem));
      } else {
        CUDA_CHECK(cudaFuncSetAttribute(k_value_to_bin_tile<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_value_to_bin_tile<double>, kVbThreads, smem));
      }
      const int64_t slots = static_cast<int64_t>(std::max(1, per_sm)) * sms;
      const int64_t col_tiles = (Fu + kVbCols - 1) / kVbCols;
      const size_t bsmem = static_cast<size_t>(kBcRows) * (Fp + 16);
      if (!direct) CUDA_CHECK(cudaFuncSetAttribute(k_bundle_columns, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bsmem)));
      for (int64_t p0 = 0; p0 < rows; p0 += piece) {
        const int64_t prow = std::min(piece, rows - p0);
        // a CTA loads its feature tile's bounds once and then walks its share of the row tiles; the grid is ONE wave of
        // resident CTAs (the tiles of a CTA are many and equal: a partial second wave would cost a whole one)
        const int64_t row_tiles = (prow + kVbRows - 1) / kVbRows;
        const int64_t gx = std::max<int64_t>(1, std::min<int64_t>(row_tiles, std::max<int64_t>(1, slots / col_tiles)));
        const dim3 tgrid(static_cast<unsigned>(gx), static_cast<unsigned>(col_tiles));
        uint8_t* o1 = direct ? dst + p0 * C : tmp_[k & 1].p;
        const int64_t pitch1 = direct ? C : Fp;
        const unsigned char* s1 = src + static_cast<size_t>(p0) * ncol * esize;
        if (dtype == 0) k_value_to_bin_tile<float><<<tgrid, kVbThreads, smem, st>>>(reinterpret_cast<const float*>(s1), ncol, static_cast<int32_t>(prow), ro, o1, pitch1, max_bounds_, max_feats_);
        else k_value_to_bin_tile<double><<<tgrid, kVbThreads, smem, st>>>(reinterpret_cast<const double*>(s1), ncol, static_cast<int32_t>(prow), ro, o1, pitch1, max_bounds_, max_feats_);
        ++launches_;
        if (!direct) {
          const unsigned g2 = static_cast<unsigned>(std::min<int64_t>((prow + kBcRows - 1) / kBcRows, static_cast<int64_t>(sms) * 8));
          k_bundle_columns<<<g2, 256, bsmem, st>>>(tmp_[k & 1].p, Fp, static_cast<int32_t>(prow), static_cast<int32_t>(Fu), d_col_first_.p, d_feat_pos_.p,
                                                  d_col_pos_.p, static_cast<int32_t>(C), dst + p0 * C, C);
          ++launches_;
        }
      }
      CUDA_CHECK(cudaGetLastError());
      if (!out_on_device) CUDA_CHECK(cudaMemcpyAsync(out + r0 * C, dst, static_cast<size_t>(rows) * C, cudaMemcpyDeviceToHost, st));
    }
    CUDA_CHECK(cudaEventRecord(ej, streams_[1]));
    CUDA_CHECK(cudaStreamWaitEvent(streams_[0], ej, 0));
    CUDA_CHECK(cudaEventRecord(e1, streams_[0]));
    CUDA_CHECK(cudaStreamSynchronize(streams_[0]));
    CUDA_CHECK(cudaStreamSynchronize(streams_[1]));
    float ms = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(ej);
    if (elapsed_ms) *elapsed_ms = ms;
  }
  int64_t launches() const { return launches_; }

 private:
  static BinFitConfig ToCfg(const LGBMB200_BinConfig& c) {
    BinFitConfig f;
    f.max_bin = c.max_bin; f.min_data_in_bin = c.min_data_in_bin; f.min_data_in_leaf = c.min_data_in_leaf;
    f.sample_cnt = c.bin_construct_sample_cnt; f.seed = c.data_random_seed;
    f.pre_filter = c.feature_pre_filter != 0; f.use_missing = c.use_missing != 0; f.zero_as_missing = c.zero_as_missing != 0;
    f.enable_bundle = c.enable_bundle != 0;
    return f;
  }
  void Upload() {
    if (uploaded_) return;
    const BinTable& t = binner_.table();
    Up(d_col_first_, t.col_first); Up(d_bounds32_, t.bounds32); Up(d_bounds64_, t.bounds64);
    Up(d_ro_real_, t.ro_feat_real); Up(d_ro_lo_, t.ro_feat_lo); Up(d_ro_num_bin_, t.ro_feat_num_bin);
    Up(d_ro_mfb_, t.ro_feat_mfb); Up(d_ro_missing_, t.ro_feat_missing); Up(d_ro_bound_first_, t.ro_bound_first); Up(d_ro_bound_count_, t.ro_bound_count);
    Up(d_feat_pos_, t.feat_pos); Up(d_col_pos_, t.col_pos);
    // shared-memory needs of k_value_to_bin_tile: the widest 32-column tile (padded, skewed bound layout: binning.cuh)
    max_bounds_ = 1; max_feats_ = 1;
    for (int p0 = 0; p0 < t.num_features; p0 += kVbCols) {            // tiles of the real-order pass: 32 features each
      const int p1 = std::min(t.num_features, p0 + kVbCols);
      max_feats_ = std::max(max_feats_, p1 - p0);
      int words = 0;
      for (int p = p0; p < p1; ++p) {
        int depth = 0;
        while ((1 << depth) - 1 < t.ro_bound_count[p]) ++depth;
        words += vb_slots(depth);
      }
      max_bounds_ = std::max(max_bounds_, words);
    }
    max_bounds_ = (max_bounds_ + 3) / 4 * 4;
    uploaded_ = true;
  }

  int device_;
  Binner binner_;
  bool fitted_ = false, uploaded_ = false;
  int max_bounds_ = 1, max_feats_ = 1;
  PinnedStager stager_;
  int64_t launches_ = 0;
  cudaStream_t streams_[2] = {nullptr, nullptr};
  DevBuf<int32_t> d_col_first_;
  DevBuf<float> d_bounds32_;
  DevBuf<double> d_bounds64_;
  DevBuf<int32_t> d_ro_real_, d_ro_lo_, d_ro_num_bin_, d_ro_mfb_, d_ro_missing_, d_ro_bound_first_, d_ro_bound_count_, d_feat_pos_, d_col_pos_;
  DevBuf<uint8_t> tmp_[2];
};

}  // namespace b200

// ---------------------------------------------------------------------------------------------------------------------
// Prediction with a trained model (SURVEY.md §8 f-4), see predict.cuh
#include "predict.cuh"

namespace b200 {

class Predictor {
 public:
  Predictor(int device, int32_t num_trees, const int32_t* tree_num_leaves, const int32_t* split_feature, const double* threshold,
            const int8_t* decision_type, const int32_t* left_child, const int32_t* right_child, const double* leaf_value,
            int32_t max_feature_idx)
      : device_(device), num_trees_(num_trees), max_feature_idx_(max_feature_idx) {
    REQUIRE(num_trees >= 0 && tree_num_leaves, "bad model");
    std::vector<PNodeA> na; std::vector<PNodeB> nb; std::vector<PNodeF> nfl; std::vector<double> leaves; std::vector<int32_t> nf, lf, nl;
    int64_t ni = 0, li = 0;
    for (int t = 0; t < num_trees; ++t) {
      const int L = tree_num_leaves[t];
      REQUIRE(L >= 1, "a tree needs at least one leaf");
      nf.push_back(static_cast<int32_t>(na.size())); lf.push_back(static_cast<int32_t>(leaves.size())); nl.push_back(L);
      for (int i = 0; i < L - 1; ++i, ++ni) {
        PNodeA a; PNodeB b;
        a.threshold = threshold[ni]; a.feature = split_feature[ni]; b.left = left_child[ni]; b.right = right_child[ni];
        // LGBM_BoosterPredictForMat reads rows through RowPairFunctionFromDenseMatrix, which drops every |x| <= kZeroThreshold
        // (c_api.cpp:2864): the tree sees 0.0 for such a value.  A threshold inside [-kZ, kZ) moved just outside the band
        // makes the plain `x <= t` of the walk equal `(|x| <= kZ ? 0.0 : x) <= t` for every x, so the kernels compare the
        // raw value and need no instruction for the band.  Bin bounds put -kZ here (bin.cpp:191,195,279).
        if (a.threshold >= -kZeroBound && a.threshold < 0.0) a.threshold = std::nextafter(-kZeroBound, -INFINITY);
        else if (a.threshold >= 0.0 && a.threshold < kZeroBound) a.threshold = kZeroBound;
        a.decision = static_cast<int32_t>(decision_type[ni]) & 0xff;
        REQUIRE(!(a.decision & 1), "categorical splits are not supported");
        REQUIRE(a.feature >= 0 && a.feature <= max_feature_idx, "split feature out of range");
        REQUIRE(b.left < L - 1 && b.right < L - 1 && ~b.left < L && ~b.right < L, "child index out of range");
        na.push_back(a); nb.push_back(b);
        REQUIRE(a.feature < (1 << 24), "feature index too large");
        PNodeF fn;
        fn.thr = static_cast<float>(a.threshold);
        if (static_cast<double>(fn.thr) > a.threshold) fn.thr = std::nextafterf(fn.thr, -INFINITY);     // the largest float <= threshold
        fn.fd = static_cast<uint32_t>(a.feature) | (static_cast<uint32_t>(a.decision) << 24); fn.left = b.left; fn.right = b.right;
        nfl.push_back(fn);
      }
      for (int i = 0; i < L; ++i, ++li) leaves.push_back(leaf_value[li]);
    }
    if (device_ >= 0) CUDA_CHECK(cudaSetDevice(device_));
    Up(d_na_, na); Up(d_nb_, nb); Up(d_nfl_, nfl); Up(d_leaves_, leaves); Up(d_nf_, nf); Up(d_lf_, lf); Up(d_nl_, nl);

    CUDA_CHECK(cudaStreamCreateWithFlags(&streams_[0], cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&streams_[1], cudaStreamNonBlocking));
  }
  ~Predictor() { for (auto& s : streams_) if (s) cudaStreamDestroy(s); }
  int device() const { return device_; }
  int64_t launches() const { return launches_; }

  // raw scores of `nrow` rows of a row-major [nrow x ncol] matrix (host: streamed in row chunks on two streams)
  void Predict(const void* data, int dtype, int64_t nrow, int32_t ncol, int data_on_device, double* out, int out_on_device, float* elapsed_ms) {
    REQUIRE(data && out && nrow > 0, "bad argument");
    REQUIRE(dtype == 0 || dtype == 1, "data_type must be 0 (float32) or 1 (float64)");
    REQUIRE(ncol > max_feature_idx_, "the matrix has fewer columns than the model's max_feature_idx + 1");
    int dev = 0;
    CUDA_CHECK(cudaGetDevice(&dev));
    const int sms = DeviceSms(dev);
    const size_t esize = dtype == 0 ? 4 : 8;
    int64_t chunk = std::max<int64_t>(1024, (static_cast<int64_t>(64) << 20) / static_cast<int64_t>(ncol * esize));
    chunk = std::min(chunk, nrow);
    if (data_on_device && out_on_device) chunk = nrow;          // nothing to stage: one launch over all rows
    DevBuf<unsigned char> dx[2]; DevBuf<double> dout[2];
    if (!data_on_device) { for (auto& b : dx) b.alloc(static_cast<size_t>(chunk) * ncol * esize); stager_.Reserve(static_cast<size_t>(chunk) * ncol * esize); }
    if (!out_on_device) for (auto& b : dout) b.alloc(static_cast<size_t>(chunk));
    const PredTable pt{d_na_.p, d_nb_.p, d_nfl_.p, d_leaves_.p, d_nf_.p, d_lf_.p, d_nl_.p, num_trees_};
    // odd row stride (in elements): 32 lanes reading one feature of 32 rows hit 32 different banks
    const int stride = ncol | 1;
    // rows per CTA tile: 64 when two such CTAs fit an SM, else 32; 0 => rows too wide to stage
    const int pass = std::getenv("LGBMB200_PRED_PASS") ? std::max(2, std::min(kPredPassMax, std::atoi(std::getenv("LGBMB200_PRED_PASS")))) : 16;      // 16 trees per pass: the nodes of a pass stay in L1
    auto tile_bytes = [&](int R) { return static_cast<size_t>(pass) * R * 8 + static_cast<size_t>(R) * stride * esize; };
    const int tile_rows = tile_bytes(64) <= 112 * 1024 ? 64 : (tile_bytes(32) <= 224 * 1024 ? 32 : 0);
    cudaEvent_t e0, e1, ej;
    CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1)); CUDA_CHECK(cudaEventCreateWithFlags(&ej, cudaEventDisableTiming));
    CUDA_CHECK(cudaDeviceSynchronize());
    CUDA_CHECK(cudaEventRecord(e0, streams_[0]));
    CUDA_CHECK(cudaStreamWaitEvent(streams_[1], e0, 0));
    int k = 0;
    for (int64_t r0 = 0; r0 < nrow; r0 += chunk, ++k) {
      const int64_t rows = std::min(chunk, nrow - r0);
      cudaStream_t st = streams_[k & 1];
      const unsigned char* src = static_cast<const unsigned char*>(data) + static_cast<size_t>(r0) * ncol * esize;
      if (!data_on_device) {
        stager_.Send(k, dx[k & 1].p, src, static_cast<size_t>(rows) * ncol * esize, st);
        src = dx[k & 1].p;
      }
      double* dst = out_on_device ? out + r0 : dout[k & 1].p;
      if (tile_rows >= 32) {
        const size_t smem = tile_bytes(tile_rows);
        int per_sm = 1;
        if (dtype == 0) {
          CUDA_CHECK(cudaFuncSetAttribute(k_predict<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
          CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_predict<float>, kPredThreads, smem));
        } else {
          CUDA_CHECK(cudaFuncSetAttribute(k_predict<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
          CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_predict<double>, kPredThreads, smem));
        }
        per_sm = std::max(1, per_sm);
        const unsigned grid = static_cast<unsigned>(std::min<int64_t>((rows + tile_rows - 1) / tile_rows, static_cast<int64_t>(sms) * per_sm));
        if (dtype == 0) {
          k_predict<float><<<grid, kPredThreads, smem, st>>>(reinterpret_cast<const float*>(src), ncol, rows, ncol, pt, dst, tile_rows, stride, pass);
        } else {
          k_predict<double><<<grid, kPredThreads, smem, st>>>(reinterpret_cast<const double*>(src), ncol, rows, ncol, pt, dst, tile_rows, stride, pass);
        }
      } else {
        const unsigned grid = static_cast<unsigned>(std::min<int64_t>((rows + kPredThreads - 1) / kPredThreads, static_cast<int64_t>(sms) * 8));
        if (dtype == 0) k_predict_wide<float><<<grid, kPredThreads, 0, st>>>(reinterpret_cast<const float*>(src), ncol, rows, pt, dst);
        else k_predict_wide<double><<<grid, kPredThreads, 0, st>>>(reinterpret_cast<const double*>(src), ncol, rows, pt, dst);
      }
      CUDA_CHECK(cudaGetLastError());
      ++launches_;
      if (!out_on_device) CUDA_CHECK(cudaMemcpyAsync(out + r0, dst, sizeof(double) * static_cast<size_t>(rows), cudaMemcpyDeviceToHost, st));
    }
    CUDA_CHECK(cudaEventRecord(ej, streams_[1]));
    CUDA_CHECK(cudaStreamWaitEvent(streams_[0], ej, 0));
    CUDA_CHECK(cudaEventRecord(e1, streams_[0]));
    CUDA_CHECK(cudaStreamSynchronize(streams_[0]));
    CUDA_CHECK(cudaStreamSynchronize(streams_[1]));
    float ms = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(ej);
    if (elapsed_ms) *elapsed_ms = ms;
  }

 private:
  int device_; int32_t num_trees_, max_feature_idx_;
  PinnedStager stager_;
  int64_t launches_ = 0;
  cudaStream_t streams_[2] = {nullptr, nullptr};
  DevBuf<PNodeA> d_na_; DevBuf<PNodeB> d_nb_; DevBuf<PNodeF> d_nfl_; DevBuf<double> d_leaves_; DevBuf<int32_t> d_nf_, d_lf_, d_nl_;
};

}  // namespace b200

// ------------------------------------------------------------------------------------------ C-ABI
using b200::CudaError;
using b200::Learner;
using b200::BinnerCtx;
using b200::Predictor;

#define API_BEGIN() try {
#define API_BEGIN_H(h) try { DeviceGuard _dev_guard((h) ? static_cast<Learner*>(h)->inited_device() : -1);
#define API_END()                                            \
  }                                                          \
  catch (const CudaError& e) { b200::g_last_error = e.msg; return -1; } \
  catch (const std::exception& e) { b200::g_last_error = e.what(); return -1; } \
  catch (...) { b200::g_last_error = "unknown error"; return -1; } \
  return 0;

// Several learners (one per GPU) may live in one process (LGBMB200_LearnersConnectLocal): every entry point runs on the
// learner's own device and restores the caller's current device afterwards.
struct DeviceGuard {
  int prev = -1; bool switched = false;
  explicit DeviceGuard(int dev) {
    if (dev >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

extern "C" {

const char* LGBMB200_GetLastError(void) { return b200::g_last_error.c_str(); }

int LGBMB200_LearnerCreate(const LGBMB200_Config* config, LGBMB200_LearnerHandle* out) {
  API_BEGIN();
  if (!config || !out) throw CudaError{"null argument"};
  *out = new Learner(*config);
  API_END();
}
int LGBMB200_LearnerInit(LGBMB200_LearnerHandle h, const LGBMB200_Layout* layout, const uint8_t* bins_host, int32_t is_constant_hessian) {
  API_BEGIN_H(h);
  if (!h || !layout || !bins_host) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->Init(*layout, bins_host, is_constant_hessian);
  API_END();
}
int LGBMB200_LearnerResetConfig(LGBMB200_LearnerHandle h, const LGBMB200_Config* config) {
  API_BEGIN_H(h);
  if (!h || !config) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->SetConfig(*config);
  API_END();
}
int LGBMB200_LearnerSetConstantHessian(LGBMB200_LearnerHandle h, int32_t is_constant_hessian) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->SetConstantHessian(is_constant_hessian);
  API_END();
}
int LGBMB200_LearnerSetFeatureMask(LGBMB200_LearnerHandle h, const uint8_t* feature_used) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->SetFeatureMask(feature_used);
  API_END();
}
int LGBMB200_LearnerSetBaggingData(LGBMB200_LearnerHandle h, const int32_t* used_indices, int32_t num_used, int32_t on_device) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->SetBagging(used_indices, num_used, on_device);
  API_END();
}
int LGBMB200_LearnerGossSample(LGBMB200_LearnerHandle h, float* grad_dev, float* hess_dev, double top_rate, double other_rate,
                               int32_t seed, int32_t iteration, int32_t* out_bag_count) {
  API_BEGIN_H(h);
  if (!h || !grad_dev || !hess_dev) throw CudaError{"null argument"};
  const int32_t n = static_cast<Learner*>(h)->GossSample(grad_dev, hess_dev, top_rate, other_rate, seed, iteration);
  if (out_bag_count) *out_bag_count = n;
  API_END();
}
int LGBMB200_LearnerGetBaggingData(LGBMB200_LearnerHandle h, int32_t* indices_host, int32_t num_indices) {
  API_BEGIN_H(h);
  if (!h || !indices_host) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->GetBag(indices_host, num_indices);
  API_END();
}
int LGBMB200_LearnerTrain(LGBMB200_LearnerHandle h, const float* gradients, const float* hessians, int32_t on_device, LGBMB200_Tree* out_tree) {
  API_BEGIN_H(h);
  if (!h || !gradients || !hessians || !out_tree) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->Train(gradients, hessians, on_device, out_tree);
  API_END();
}
int LGBMB200_LearnerAddPredictionToScore(LGBMB200_LearnerHandle h, const double* leaf_value, int32_t num_leaves, double* score, int32_t on_device) {
  API_BEGIN_H(h);
  if (!h || !leaf_value || !score) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->AddPredictionToScore(leaf_value, num_leaves, score, on_device);
  API_END();
}
int LGBMB200_LearnerAddPredictionAllRows(LGBMB200_LearnerHandle h, const double* leaf_value, int32_t num_leaves, double* score_dev) {
  API_BEGIN_H(h);
  if (!h || !leaf_value || !score_dev) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->RouteAllRows(leaf_value, num_leaves, score_dev, nullptr);
  API_END();
}
int LGBMB200_LearnerGetPartition(LGBMB200_LearnerHandle h, int32_t* leaf_begin, int32_t* leaf_count, int32_t* indices) {
  API_BEGIN_H(h);
  if (!h || !leaf_begin || !leaf_count || !indices) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->GetPartition(leaf_begin, leaf_count, indices);
  API_END();
}
int LGBMB200_LearnerGetLeafHistogram(LGBMB200_LearnerHandle h, int32_t leaf, double* out) {
  API_BEGIN_H(h);
  if (!h || !out) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->GetLeafHistogram(leaf, out);
  API_END();
}
int LGBMB200_LearnerConstructHistogram(LGBMB200_LearnerHandle h, const float* gradients, const float* hessians, int32_t on_device,
                                       const int32_t* indices_host, int32_t num_indices, double* hist_out, float* elapsed_ms) {
  API_BEGIN_H(h);
  if (!h || !gradients || !hessians) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->ConstructHistogram(gradients, hessians, on_device, indices_host, num_indices, hist_out, elapsed_ms);
  API_END();
}
int LGBMB200_L2Gradients(LGBMB200_LearnerHandle h, const double* score_dev, const float* label_dev, float* grad_dev, float* hess_dev, int32_t n) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->L2Gradients(score_dev, label_dev, grad_dev, hess_dev, n);
  API_END();
}
int LGBMB200_BinaryGradients(LGBMB200_LearnerHandle h, const double* score_dev, const float* label_dev, float* grad_dev, float* hess_dev,
                             int32_t n, double sigmoid) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->BinaryGradients(score_dev, label_dev, grad_dev, hess_dev, n, sigmoid);
  API_END();
}
int64_t LGBMB200_LearnerKernelLaunches(LGBMB200_LearnerHandle h) { return h ? static_cast<Learner*>(h)->launches() : 0; }
int LGBMB200_LearnerHistStats(LGBMB200_LearnerHandle h, int32_t reset, double* hist_ms, double* hist_rows, int64_t* hist_launches) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->HistStats(reset, hist_ms, hist_rows, hist_launches);
  API_END();
}
int LGBMB200_LearnerProfileByKind(LGBMB200_LearnerHandle h, double* ms_out_9) {
  API_BEGIN_H(h);
  if (!h || !ms_out_9) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->ProfileByKind(ms_out_9);
  API_END();
}
int LGBMB200_LearnerSetProfiling(LGBMB200_LearnerHandle h, int32_t enable) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->SetProfiling(enable);
  API_END();
}
int LGBMB200_LearnerCommExport(LGBMB200_LearnerHandle h, uint8_t* handle_out_64) {
  API_BEGIN_H(h);
  if (!h || !handle_out_64) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->CommExport(handle_out_64);
  API_END();
}
int LGBMB200_LearnerCommConnect(LGBMB200_LearnerHandle h, int32_t rank, int32_t world, const uint8_t* all_handles,
                                const int32_t* feature_offsets) {
  API_BEGIN_H(h);
  if (!h || !all_handles || !feature_offsets) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->CommConnect(rank, world, all_handles, feature_offsets);
  API_END();
}
// Feature-shard bootstrap for `world` learners that live in ONE process, one per GPU (the reference's own multi-GPU
// shape: one host thread per device, include/LightGBM/cuda/cuda_nccl_topology.hpp:177-188): peer access instead of CUDA
// IPC.  handles[r] = the learner of rank r, already Init-ed with its column slice.
int LGBMB200_LearnersConnectLocal(LGBMB200_LearnerHandle* handles, int32_t world, const int32_t* feature_offsets, int32_t replicate_columns) {
  API_BEGIN();
  if (!handles || !feature_offsets || world < 1 || world > b200::kMaxRanks) throw CudaError{"bad argument"};
  int prev = 0;
  CUDA_CHECK(cudaGetDevice(&prev));
  std::vector<Learner*> L(world);
  std::vector<void*> blocks(world);
  for (int r = 0; r < world; ++r) {
    if (!handles[r]) throw CudaError{"null learner"};
    L[r] = static_cast<Learner*>(handles[r]);
    CUDA_CHECK(cudaSetDevice(L[r]->device()));
    blocks[r] = L[r]->CommPrepare();
  }
  for (int i = 0; i < world; ++i) {
    CUDA_CHECK(cudaSetDevice(L[i]->device()));
    for (int j = 0; j < world; ++j) {
      if (L[j]->device() == L[i]->device()) continue;
      const cudaError_t e = cudaDeviceEnablePeerAccess(L[j]->device(), 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      else if (e != cudaSuccess) { cudaSetDevice(prev); throw CudaError{std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e)}; }
    }
  }
  for (int r = 0; r < world; ++r) {
    CUDA_CHECK(cudaSetDevice(L[r]->device()));
    L[r]->CommConnectPtrs(r, world, blocks.data(), feature_offsets);
  }
  if (replicate_columns && world > 1) {
    std::vector<const uint8_t*> cols(world);
    for (int r = 0; r < world; ++r) cols[r] = L[r]->ColumnsPtr();
    for (int r = 0; r < world; ++r) {
      CUDA_CHECK(cudaSetDevice(L[r]->device()));
      L[r]->CommShareColumnsPtrs(cols.data());
    }
  }
  CUDA_CHECK(cudaSetDevice(prev));
  API_END();
}
int LGBMB200_LearnerCommExportColumns(LGBMB200_LearnerHandle h, uint8_t* handle_out_64) {
  API_BEGIN_H(h);
  REQUIRE(h && handle_out_64, "null argument");
  static_cast<Learner*>(h)->CommExportColumns(handle_out_64);
  API_END();
}
int LGBMB200_LearnerCommShareColumns(LGBMB200_LearnerHandle h, const uint8_t* all_column_handles) {
  API_BEGIN_H(h);
  REQUIRE(h && all_column_handles, "null argument");
  static_cast<Learner*>(h)->CommShareColumns(all_column_handles);
  API_END();
}
int LGBMB200_LearnerCommExportPool(LGBMB200_LearnerHandle h, uint8_t* handle_out_64) {
  API_BEGIN_H(h);
  if (!h || !handle_out_64) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->CommExportPool(handle_out_64);
  API_END();
}
int LGBMB200_LearnerCommConnectRows(LGBMB200_LearnerHandle h, int32_t rank, int32_t world, const uint8_t* comm_handles,
                                    const uint8_t* pool_handles) {
  API_BEGIN_H(h);
  if (!h || !comm_handles || !pool_handles) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->CommConnectRows(rank, world, comm_handles, pool_handles);
  API_END();
}
int LGBMB200_LearnerGetLeafIndex(LGBMB200_LearnerHandle h, int32_t* leaf_index_host) {
  API_BEGIN_H(h);
  if (!h || !leaf_index_host) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->GetLeafIndex(leaf_index_host);
  API_END();
}
int LGBMB200_LearnerGetLeafIndexRange8(LGBMB200_LearnerHandle h, int32_t row_lo, int32_t row_hi, uint8_t* leaf_index_host) {
  API_BEGIN_H(h);
  if (!h || !leaf_index_host) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->GetLeafIndexRange8(row_lo, row_hi, leaf_index_host);
  API_END();
}
int LGBMB200_LearnerTimerStart(LGBMB200_LearnerHandle h) {
  API_BEGIN_H(h);
  if (!h) throw CudaError{"null argument"};
  static_cast<Learner*>(h)->TimerStart();
  API_END();
}
int LGBMB200_LearnerTimerStop(LGBMB200_LearnerHandle h, float* elapsed_ms) {
  API_BEGIN_H(h);
  if (!h || !elapsed_ms) throw CudaError{"null argument"};
  *elapsed_ms = static_cast<Learner*>(h)->TimerStop();
  API_END();
}
int LGBMB200_HostAllocPinned(void** ptr, int64_t bytes) {
  API_BEGIN();
  if (!ptr) throw CudaError{"null argument"};
  CUDA_CHECK(cudaMallocHost(ptr, static_cast<size_t>(bytes > 0 ? bytes : 1)));
  API_END();
}
int LGBMB200_HostFreePinned(void* ptr) {
  API_BEGIN();
  CUDA_CHECK(cudaFreeHost(ptr));
  API_END();
}
int LGBMB200_DeviceAlloc(void** ptr, int64_t bytes) {
  API_BEGIN();
  if (!ptr) throw CudaError{"null argument"};
  CUDA_CHECK(cudaMalloc(ptr, static_cast<size_t>(bytes > 0 ? bytes : 1)));
  API_END();
}
int LGBMB200_DeviceFree(void* ptr) {
  API_BEGIN();
  CUDA_CHECK(cudaFree(ptr));
  API_END();
}
int LGBMB200_MemcpyH2D(void* dst_dev, const void* src_host, int64_t bytes) {
  API_BEGIN();
  CUDA_CHECK(cudaMemcpy(dst_dev, src_host, static_cast<size_t>(bytes), cudaMemcpyHostToDevice));
  API_END();
}
int LGBMB200_MemcpyD2H(void* dst_host, const void* src_dev, int64_t bytes) {
  API_BEGIN();
  CUDA_CHECK(cudaMemcpy(dst_host, src_dev, static_cast<size_t>(bytes), cudaMemcpyDeviceToHost));
  API_END();
}
int LGBMB200_LearnerFree(LGBMB200_LearnerHandle h) {
  API_BEGIN_H(h);
  delete static_cast<Learner*>(h);
  API_END();
}

// ---- Dataset construction (binning.cuh)
int LGBMB200_BinnerCreate(const LGBMB200_BinConfig* config, LGBMB200_BinnerHandle* out) {
  API_BEGIN();
  if (!config || !out) throw CudaError{"null argument"};
  *out = new BinnerCtx(*config);
  API_END();
}
int LGBMB200_BinnerFit(LGBMB200_BinnerHandle h, const void* data, int32_t data_type, int32_t nrow, int32_t ncol, int32_t is_row_major) {
  API_BEGIN();
  if (!h) throw CudaError{"null argument"};
  static_cast<BinnerCtx*>(h)->Fit(data, data_type, nrow, ncol, is_row_major);
  API_END();
}
int LGBMB200_BinnerGetLayout(LGBMB200_BinnerHandle h, LGBMB200_Layout* out) {
  API_BEGIN();
  if (!h || !out) throw CudaError{"null argument"};
  static_cast<const BinnerCtx*>(h)->GetLayout(out);
  API_END();
}
int LGBMB200_BinnerGetFeatureBounds(LGBMB200_BinnerHandle h, int32_t inner_feature, double* upper_bounds_out, int32_t* num_bin_out) {
  API_BEGIN();
  if (!h) throw CudaError{"null argument"};
  static_cast<const BinnerCtx*>(h)->GetBounds(inner_feature, upper_bounds_out, num_bin_out);
  API_END();
}
int LGBMB200_BinnerGetSampleIndices(LGBMB200_BinnerHandle h, int32_t* indices_out, int32_t* num_out) {
  API_BEGIN();
  if (!h || !num_out) throw CudaError{"null argument"};
  *num_out = static_cast<const BinnerCtx*>(h)->GetSampleRows(indices_out);
  API_END();
}
int LGBMB200_BinnerTransform(LGBMB200_BinnerHandle h, const void* data, int32_t data_type, int32_t nrow, int32_t data_on_device,
                             uint8_t* bins_out, int32_t out_on_device, float* elapsed_ms) {
  API_BEGIN();
  if (!h) throw CudaError{"null argument"};
  DeviceGuard guard(static_cast<BinnerCtx*>(h)->device());
  static_cast<BinnerCtx*>(h)->Transform(data, data_type, nrow, data_on_device, bins_out, out_on_device, elapsed_ms);
  API_END();
}
int LGBMB200_BinnerFree(LGBMB200_BinnerHandle h) {
  API_BEGIN();
  if (h) { DeviceGuard guard(static_cast<BinnerCtx*>(h)->device()); delete static_cast<BinnerCtx*>(h); }
  API_END();
}

// ---- Prediction (predict.cuh)
int LGBMB200_PredictorCreate(int32_t gpu_device_id, int32_t num_trees, const int32_t* tree_num_leaves, const int32_t* split_feature,
                             const double* threshold, const int8_t* decision_type, const int32_t* left_child, const int32_t* right_child,
                             const double* leaf_value, int32_t max_feature_idx, LGBMB200_PredictorHandle* out) {
  API_BEGIN();
  if (!out) throw CudaError{"null argument"};
  DeviceGuard guard(gpu_device_id);
  *out = new Predictor(gpu_device_id, num_trees, tree_num_leaves, split_feature, threshold, decision_type, left_child, right_child,
                       leaf_value, max_feature_idx);
  API_END();
}
int LGBMB200_PredictorPredict(LGBMB200_PredictorHandle h, const void* data, int32_t data_type, int32_t nrow, int32_t ncol,
                              int32_t data_on_device, double* out_raw_score, int32_t out_on_device, float* elapsed_ms) {
  API_BEGIN();
  if (!h) throw CudaError{"null argument"};
  DeviceGuard guard(static_cast<Predictor*>(h)->device());
  static_cast<Predictor*>(h)->Predict(data, data_type, nrow, ncol, data_on_device, out_raw_score, out_on_device, elapsed_ms);
  API_END();
}
int LGBMB200_PredictorFree(LGBMB200_PredictorHandle h) {
  API_BEGIN();
  if (h) { DeviceGuard guard(static_cast<Predictor*>(h)->device()); delete static_cast<Predictor*>(h); }
  API_END();
}

}  // extern "C"
