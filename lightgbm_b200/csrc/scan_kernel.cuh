// scan_kernel.cuh — FixHistogram + histogram subtraction + split-gain scan, fused (sm_90a).
//
// Replaces: Dataset::FixHistogram (reference src/io/dataset.cpp:1519-1537), FeatureHistogram::Subtract
// (src/treelearner/feature_histogram.hpp:96-145), FeatureHistogram::FindBestThreshold ->
// FindBestThresholdSequentially (feature_histogram.hpp:165-175, :830-1057) and the per-leaf arg-max of
// SerialTreeLearner::FindBestSplitsFromHistograms (src/treelearner/serial_tree_learner.cpp:480-624).
//
// One warp per feature handles BOTH children of the last split: it loads the smaller child's slice
// (<=256 bins, 8 per lane), fixes the most-frequent-bin entry, scans it, then forms
// larger = parent - smaller in exact int64 arithmetic (written back in place into the parent's pool
// slot, which becomes the larger child's) and scans that.  The sequential right->left / left->right
// accumulation of the reference becomes: lane-local totals -> 5-step warp shuffle scan of lane
// offsets -> lane-local sequential pass evaluating candidates -> warp arg-max with the reference's
// tie-break (first candidate in scan order wins, strict '>').
//
// Tie consistency: in the reference two thresholds separated by an EMPTY bin give bit-identical sums
// and the first in scan order wins.  A parallel prefix is not bit-consistent across lanes, so the
// rule is applied explicitly: a candidate whose just-accumulated bin is empty is a duplicate of the
// previous candidate and is skipped.  With the int64 pool an empty bin is exactly (0,0).  A bin whose rows all have
// hessian 0 (a saturated logistic) is (g, 0) with g != 0: it is not empty, and its gradient counts like any other.
#pragma once
#include "comm.cuh"
#include "types.cuh"

namespace b200 {

struct GainCfg {
  int use_l1, use_max_output, use_smoothing;
  double l1, l2, max_delta_step, smoothing;
};

__device__ __forceinline__ GainCfg make_gain_cfg(const Params& P) {
  GainCfg c;
  c.use_l1 = P.l1 > 0.0;
  c.use_max_output = P.max_delta_step > 0.0;
  c.use_smoothing = P.path_smooth > B200_KEPS;
  c.l1 = P.l1; c.l2 = P.l2; c.max_delta_step = P.max_delta_step; c.smoothing = P.path_smooth;
  return c;
}

__device__ __forceinline__ double sign_of(double x) { return static_cast<double>((x > 0.0) - (x < 0.0)); }

// feature_histogram.hpp:711-714
__device__ __forceinline__ double threshold_l1(double s, double l1) {
  double r = fabs(s) - l1;
  if (r < 0.0) r = 0.0;
  return sign_of(s) * r;
}

// NOTE on code size: the first version of k_scan inlined the fp64 divisions of the gain formula ~100 times
// (26K SASS instructions = 416 KB) and spent most of its time waiting for instruction fetch.  The gain helpers are therefore
// real functions (__noinline__), called from a single scan site per direction.
// feature_histogram.hpp:716-738 CalculateSplittedLeafOutput (no monotone constraints)
__device__ __noinline__ double leaf_output(const GainCfg& c, double sg, double sh, int n, double parent_output) {
  double ret = c.use_l1 ? -threshold_l1(sg, c.l1) / (sh + c.l2) : -sg / (sh + c.l2);
  if (c.use_max_output) {
    if (c.max_delta_step > 0 && fabs(ret) > c.max_delta_step) ret = sign_of(ret) * c.max_delta_step;
  }
  if (c.use_smoothing) {
    const double w = n / c.smoothing;
    ret = ret * w / (w + 1) + parent_output / (w + 1);
  }
  return ret;
}

// feature_histogram.hpp:799-828 GetLeafGain / GetLeafGainGivenOutput
__device__ __noinline__ double leaf_gain(const GainCfg& c, double sg, double sh, int n, double parent_output) {
  const double g = c.use_l1 ? threshold_l1(sg, c.l1) : sg;
  if (!c.use_max_output && !c.use_smoothing) return (g * g) / (sh + c.l2);
  const double out = leaf_output(c, sg, sh, n, parent_output);
  return -(2.0 * g * out + (sh + c.l2) * out * out);
}

// GetSplitGains (feature_histogram.hpp:758-797, no monotone constraints): left + right leaf gains
__device__ __noinline__ double split_gain(const GainCfg& c, double lg, double lh, int lc, double rg, double rh, int rc, double parent_output) {
  if (!c.use_l1 && !c.use_max_output && !c.use_smoothing) return (lg * lg) / (lh + c.l2) + (rg * rg) / (rh + c.l2);
  return leaf_gain(c, lg, lh, lc, parent_output) + leaf_gain(c, rg, rh, rc, parent_output);
}

__device__ __forceinline__ double shfl_down_d(double v, int d) { return __shfl_down_sync(0xffffffffu, v, d); }
__device__ __forceinline__ double shfl_up_d(double v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }

struct DirBest {
  double gain, slg, slh;
  int threshold, left_count, pos;   // pos: rank in scan order (smaller = earlier)
};

// One scan direction over the lane's 8 slice entries g[k], h[k] (entry e = lane*8+k <-> bin e+offset).
// Returns the warp-wide best candidate (all lanes hold the same result); *any_splittable is OR-ed.
template <bool REVERSE>
__device__ __noinline__ DirBest scan_direction(const double (&g)[8], const double (&h)[8], int lane, const FeatMeta& m,
                                                  const Params& P, const GainCfg& gc, double sum_g, double sum_h,
                                                  int num_data, double min_gain_shift, double parent_output,
                                                  bool skip_default, bool na_as_missing, int* any_splittable) {
  const double cnt_factor = num_data / sum_h;
  const int nslice = m.nslice, offset = m.offset;
  // entries that take part in the accumulation (feature_histogram.hpp:861-867 / :964-970)
  int e_lo, e_hi;
  if (REVERSE) { e_lo = 1 - offset; e_hi = nslice - 1 - (na_as_missing ? 1 : 0); }
  else { e_lo = 0; e_hi = m.num_bin - 2 - offset; }
  const int skip_e = skip_default ? (m.default_bin - offset) : -1000;

  // pass 1: lane totals
  double tg = 0.0, th = 0.0; int tc = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int e = lane * 8 + k;
    if (e >= e_lo && e <= e_hi && e != skip_e) { tg += g[k]; th += h[k]; tc += static_cast<int>(h[k] * cnt_factor + 0.5); }
  }
  // inclusive scan of lane totals in scan order (REVERSE: lanes above me come first), then shift by one
  double og = tg, oh = th; int oc = tc;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    if (REVERSE) {
      const double xg = shfl_down_d(og, d), xh = shfl_down_d(oh, d); const int xc = __shfl_down_sync(0xffffffffu, oc, d);
      if (lane + d < 32) { og += xg; oh += xh; oc += xc; }
    } else {
      const double xg = shfl_up_d(og, d), xh = shfl_up_d(oh, d); const int xc = __shfl_up_sync(0xffffffffu, oc, d);
      if (lane >= d) { og += xg; oh += xh; oc += xc; }
    }
  }
  {
    const double ig = REVERSE ? shfl_down_d(og, 1) : shfl_up_d(og, 1);
    const double ih = REVERSE ? shfl_down_d(oh, 1) : shfl_up_d(oh, 1);
    const int ic = REVERSE ? __shfl_down_sync(0xffffffffu, oc, 1) : __shfl_up_sync(0xffffffffu, oc, 1);
    const bool first = REVERSE ? (lane == 31) : (lane == 0);
    og = first ? 0.0 : ig; oh = first ? 0.0 : ih; oc = first ? 0 : ic;
  }

  // running sums at the start of this lane's entries
  double ag, ah; int ac;
  if (REVERSE) { ag = og; ah = B200_KEPS + oh; ac = oc; }
  else {
    ag = og; ah = B200_KEPS + oh; ac = oc;
    if (na_as_missing && offset == 1) {
      // implicit bin 0 = total - sum(all slice entries) (feature_histogram.hpp:945-961)
      double ag_all = 0.0, ah_all = 0.0; int ac_all = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int e = lane * 8 + k;
        if (e < nslice) { ag_all += g[k]; ah_all += h[k]; ac_all += static_cast<int>(h[k] * cnt_factor + 0.5); }
      }
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) {
        ag_all += __shfl_xor_sync(0xffffffffu, ag_all, d);
        ah_all += __shfl_xor_sync(0xffffffffu, ah_all, d);
        ac_all += __shfl_xor_sync(0xffffffffu, ac_all, d);
      }
      ag = (sum_g - ag_all) + og;
      ah = ((sum_h - B200_KEPS) - ah_all) + oh;
      ac = (num_data - ac_all) + oc;
    }
  }

  DirBest best; best.gain = -INFINITY; best.slg = 0; best.slh = 0; best.threshold = 0; best.left_count = 0; best.pos = 0x7fffffff;
  int splittable = 0;

  auto evaluate = [&](double acc_g, double acc_h, int acc_c, int threshold, int pos) {
    // acc_* are the sums of the side being accumulated (right for REVERSE, left for forward)
    if (acc_c < P.min_data_in_leaf || acc_h < P.min_sum_hessian) return;
    const int other_c = num_data - acc_c;
    if (other_c < P.min_data_in_leaf) return;
    const double other_h = sum_h - acc_h;
    if (other_h < P.min_sum_hessian) return;
    const double other_g = sum_g - acc_g;
    const double cur = REVERSE ? split_gain(gc, other_g, other_h, other_c, acc_g, acc_h, acc_c, parent_output)
                               : split_gain(gc, acc_g, acc_h, acc_c, other_g, other_h, other_c, parent_output);
    if (cur <= min_gain_shift) return;
    splittable = 1;
    if (cur > best.gain) {
      best.gain = cur; best.threshold = threshold; best.pos = pos;
      if (REVERSE) { best.slg = other_g; best.slh = other_h; best.left_count = other_c; }
      else { best.slg = acc_g; best.slh = acc_h; best.left_count = acc_c; }
    }
  };

  if (!REVERSE && na_as_missing && offset == 1 && lane == 0) {
    // the t = -1 candidate: only the implicit bin 0 on the left (threshold 0)
    evaluate(ag, ah, ac, 0, -1);
  }
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const int k = REVERSE ? 7 - kk : kk;
    const int e = lane * 8 + k;
    if (e >= e_lo && e <= e_hi && e != skip_e) {
      ag += g[k]; ah += h[k]; ac += static_cast<int>(h[k] * cnt_factor + 0.5);
      // duplicate-of-previous rule: an empty bin does not create a new candidate
      const bool empty = (g[k] == 0.0 && h[k] == 0.0);
      if (!empty) {
        if (REVERSE) evaluate(ag, ah, ac, e - 1 + offset, 255 - e);
        else evaluate(ag, ah, ac, e + offset, e);
      }
    }
  }

  // warp arg-max: larger gain, then earlier scan position
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    const double og2 = __shfl_xor_sync(0xffffffffu, best.gain, d);
    const int op = __shfl_xor_sync(0xffffffffu, best.pos, d);
    const double oslg = __shfl_xor_sync(0xffffffffu, best.slg, d);
    const double oslh = __shfl_xor_sync(0xffffffffu, best.slh, d);
    const int ot = __shfl_xor_sync(0xffffffffu, best.threshold, d);
    const int olc = __shfl_xor_sync(0xffffffffu, best.left_count, d);
    if (og2 > best.gain || (og2 == best.gain && op < best.pos)) {
      best.gain = og2; best.pos = op; best.slg = oslg; best.slh = oslh; best.threshold = ot; best.left_count = olc;
    }
  }
  if (__any_sync(0xffffffffu, splittable)) *any_splittable = 1;
  return best;
}

// FeatureHistogram::FindBestThreshold for one feature; all lanes return the same Cand.
__device__ __forceinline__ Cand find_best_threshold(const double (&g)[8], const double (&h)[8], int lane, int f,
                                                    const FeatMeta& m, const Params& P, const GainCfg& gc,
                                                    double sum_g, double sum_h_in, int num_data, double parent_output,
                                                    int* is_splittable) {
  Cand out;
  out.gain = -INFINITY; out.feature = f; out.threshold = 0; out.default_left = 1;
  out.lsg = out.lsh = out.lout = out.rsg = out.rsh = out.rout = 0.0; out.left_count = out.right_count = 0; out.pad = 0;
  out.real = m.real_index; out.owner = 0; out.ilg = 0; out.ilh = 0;
  const double sum_h = sum_h_in + 2 * B200_KEPS;
  const double min_gain_shift = leaf_gain(gc, sum_g, sum_h, num_data, parent_output) + P.min_gain_to_split;
  int splittable = 0;

  auto apply = [&](const DirBest& b, bool reverse) {
    // feature_histogram.hpp:1031-1056
    if (splittable && b.gain > out.gain + min_gain_shift) {
      out.threshold = b.threshold;
      out.lout = leaf_output(gc, b.slg, b.slh, b.left_count, parent_output);
      out.left_count = b.left_count;
      out.lsg = b.slg;
      out.lsh = b.slh - B200_KEPS;
      out.rout = leaf_output(gc, sum_g - b.slg, sum_h - b.slh, num_data - b.left_count, parent_output);
      out.right_count = num_data - b.left_count;
      out.rsg = sum_g - b.slg;
      out.rsh = sum_h - b.slh - B200_KEPS;
      out.gain = b.gain - min_gain_shift;
      out.default_left = reverse ? 1 : 0;
    }
  };

  // direction dispatch: feature_histogram.hpp:396-441 (one call site per direction keeps the kernel small)
  const bool two_way = m.num_bin > 2 && m.missing != 0;
  const bool zero = two_way && m.missing == 1, na = two_way && m.missing == 2;
  {
    const DirBest r = scan_direction<true>(g, h, lane, m, P, gc, sum_g, sum_h, num_data, min_gain_shift, parent_output, zero, na, &splittable);
    apply(r, true);
  }
  if (two_way) {
    const DirBest fw = scan_direction<false>(g, h, lane, m, P, gc, sum_g, sum_h, num_data, min_gain_shift, parent_output, zero, na, &splittable);
    apply(fw, false);
  } else if (m.missing == 2) {
    out.default_left = 0;
  }
  *is_splittable = splittable;
  return out;
}

// ---------------------------------------------------------------------------------------------------
// Quantized-gradient training: FindBestThresholdSequentiallyInt (feature_histogram.hpp:1059-1350).  The histogram
// entries are exact integer sums; the reference packs (gradient << bits | hessian) into one integer with 16- or
// 32-bit fields chosen per leaf so that nothing overflows, i.e. plain integer arithmetic on the two sums, done here
// on separate int64 values.  Doubles appear only at the candidate evaluation: sum * grad_scale / hess_scale, counts
// RoundInt(int_hessian * num_data / int_sum_hessian), kEpsilon added to the hessians at the gain call only.
struct DirBestInt {
  double gain;
  long long ilg, ilh;
  int threshold, pos;
};

template <bool REVERSE>
__device__ __noinline__ DirBestInt scan_direction_int(const long long (&g)[8], const long long (&h)[8], int lane, const FeatMeta& m,
                                                      const Params& P, const GainCfg& gc, long long tot_g, long long tot_h,
                                                      double gscale, double hscale, int num_data, double min_gain_shift,
                                                      double parent_output, bool skip_default, bool na_as_missing, int* any_splittable) {
  const double cnt_factor = static_cast<double>(num_data) / static_cast<double>(static_cast<unsigned>(tot_h));
  const int nslice = m.nslice, offset = m.offset;
  int e_lo, e_hi;
  if (REVERSE) { e_lo = 1 - offset; e_hi = nslice - 1 - (na_as_missing ? 1 : 0); }
  else { e_lo = 0; e_hi = m.num_bin - 2 - offset; }
  const int skip_e = skip_default ? (m.default_bin - offset) : -1000;

  long long tg = 0, th = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int e = lane * 8 + k;
    if (e >= e_lo && e <= e_hi && e != skip_e) { tg += g[k]; th += h[k]; }
  }
  long long og = tg, oh = th;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    if (REVERSE) {
      const long long xg = __shfl_down_sync(0xffffffffu, og, d), xh = __shfl_down_sync(0xffffffffu, oh, d);
      if (lane + d < 32) { og += xg; oh += xh; }
    } else {
      const long long xg = __shfl_up_sync(0xffffffffu, og, d), xh = __shfl_up_sync(0xffffffffu, oh, d);
      if (lane >= d) { og += xg; oh += xh; }
    }
  }
  {
    const long long ig = REVERSE ? __shfl_down_sync(0xffffffffu, og, 1) : __shfl_up_sync(0xffffffffu, og, 1);
    const long long ih = REVERSE ? __shfl_down_sync(0xffffffffu, oh, 1) : __shfl_up_sync(0xffffffffu, oh, 1);
    const bool first = REVERSE ? (lane == 31) : (lane == 0);
    og = first ? 0 : ig; oh = first ? 0 : ih;
  }
  long long ag = og, ah = oh;
  if (!REVERSE && na_as_missing && offset == 1) {
    // implicit bin 0 = total - sum(all slice entries) (feature_histogram.hpp:1196-1214)
    long long ag_all = 0, ah_all = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { if (lane * 8 + k < nslice) { ag_all += g[k]; ah_all += h[k]; } }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) { ag_all += __shfl_xor_sync(0xffffffffu, ag_all, d); ah_all += __shfl_xor_sync(0xffffffffu, ah_all, d); }
    ag = (tot_g - ag_all) + og;
    ah = (tot_h - ah_all) + oh;
  }

  DirBestInt best; best.gain = -INFINITY; best.ilg = 0; best.ilh = 0; best.threshold = 0; best.pos = 0x7fffffff;
  int splittable = 0;

  auto evaluate = [&](long long acc_g, long long acc_h, int threshold, int pos) {
    const int acc_c = static_cast<int>(static_cast<double>(static_cast<unsigned>(acc_h)) * cnt_factor + 0.5);
    const double acc_hd = static_cast<double>(static_cast<unsigned>(acc_h)) * hscale;
    if (acc_c < P.min_data_in_leaf || acc_hd < P.min_sum_hessian) return;
    const int other_c = num_data - acc_c;
    if (other_c < P.min_data_in_leaf) return;
    const long long oth_g = tot_g - acc_g, oth_h = tot_h - acc_h;
    const double other_hd = static_cast<double>(static_cast<unsigned>(oth_h)) * hscale;
    if (other_hd < P.min_sum_hessian) return;
    const double acc_gd = static_cast<double>(acc_g) * gscale, other_gd = static_cast<double>(oth_g) * gscale;
    const double cur = REVERSE ? split_gain(gc, other_gd, other_hd + B200_KEPS, other_c, acc_gd, acc_hd + B200_KEPS, acc_c, parent_output)
                               : split_gain(gc, acc_gd, acc_hd + B200_KEPS, acc_c, other_gd, other_hd + B200_KEPS, other_c, parent_output);
    if (cur <= min_gain_shift) return;
    splittable = 1;
    if (cur > best.gain) {
      best.gain = cur; best.threshold = threshold; best.pos = pos;
      if (REVERSE) { best.ilg = oth_g; best.ilh = oth_h; } else { best.ilg = acc_g; best.ilh = acc_h; }
    }
  };

  if (!REVERSE && na_as_missing && offset == 1 && lane == 0) evaluate(ag, ah, 0, -1);
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const int k = REVERSE ? 7 - kk : kk;
    const int e = lane * 8 + k;
    if (e >= e_lo && e <= e_hi && e != skip_e) {
      ag += g[k]; ah += h[k];
      // an empty bin leaves the sums unchanged: the candidate is a bit-identical duplicate of the previous one,
      // which wins the reference's strict '>' — skip it
      if (g[k] != 0 || h[k] != 0) {
        if (REVERSE) evaluate(ag, ah, e - 1 + offset, 255 - e);
        else evaluate(ag, ah, e + offset, e);
      }
    }
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    const double og2 = __shfl_xor_sync(0xffffffffu, best.gain, d);
    const int op = __shfl_xor_sync(0xffffffffu, best.pos, d);
    const long long oilg = __shfl_xor_sync(0xffffffffu, best.ilg, d);
    const long long oilh = __shfl_xor_sync(0xffffffffu, best.ilh, d);
    const int ot = __shfl_xor_sync(0xffffffffu, best.threshold, d);
    if (og2 > best.gain || (og2 == best.gain && op < best.pos)) {
      best.gain = og2; best.pos = op; best.ilg = oilg; best.ilh = oilh; best.threshold = ot;
    }
  }
  if (__any_sync(0xffffffffu, splittable)) *any_splittable = 1;
  return best;
}

// FeatureHistogram::FindBestThresholdInt (:176-189) + BeforeNumericalInt (:209-228) + output (:1303-1346)
__device__ __forceinline__ Cand find_best_threshold_int(const long long (&g)[8], const long long (&h)[8], int lane, int f,
                                                        const FeatMeta& m, const Params& P, const GainCfg& gc,
                                                        long long tot_g, long long tot_h, double gscale, double hscale,
                                                        int num_data, double parent_output, int* is_splittable) {
  Cand out;
  out.gain = -INFINITY; out.feature = f; out.threshold = 0; out.default_left = 1;
  out.lsg = out.lsh = out.lout = out.rsg = out.rsh = out.rout = 0.0; out.left_count = out.right_count = 0; out.pad = 0;
  out.real = m.real_index; out.owner = 0; out.ilg = 0; out.ilh = 0;
  const double sum_g = static_cast<double>(static_cast<int>(tot_g)) * gscale;
  const double sum_h = static_cast<double>(static_cast<unsigned>(tot_h)) * hscale;
  const double min_gain_shift = leaf_gain(gc, sum_g, sum_h, num_data, parent_output) + P.min_gain_to_split;
  const double cnt_factor = static_cast<double>(num_data) / static_cast<double>(static_cast<unsigned>(tot_h));
  int splittable = 0;

  auto apply = [&](const DirBestInt& b, bool reverse) {
    if (splittable && b.gain > out.gain + min_gain_shift) {
      const long long irg = tot_g - b.ilg, irh = tot_h - b.ilh;
      const double slg = static_cast<double>(b.ilg) * gscale, slh = static_cast<double>(static_cast<unsigned>(b.ilh)) * hscale;
      const double srg = static_cast<double>(irg) * gscale, srh = static_cast<double>(static_cast<unsigned>(irh)) * hscale;
      const int lc = static_cast<int>(static_cast<double>(static_cast<unsigned>(b.ilh)) * cnt_factor + 0.5);
      const int rc = static_cast<int>(static_cast<double>(static_cast<unsigned>(irh)) * cnt_factor + 0.5);
      out.threshold = b.threshold;
      out.lout = leaf_output(gc, slg, slh, lc, parent_output);
      out.left_count = lc; out.lsg = slg; out.lsh = slh;
      out.rout = leaf_output(gc, srg, srh, rc, parent_output);
      out.right_count = rc; out.rsg = srg; out.rsh = srh;
      out.ilg = b.ilg; out.ilh = b.ilh;
      out.gain = b.gain - min_gain_shift;
      out.default_left = reverse ? 1 : 0;
    }
  };

  const bool two_way = m.num_bin > 2 && m.missing != 0;
  const bool zero = two_way && m.missing == 1, na = two_way && m.missing == 2;
  {
    const DirBestInt r = scan_direction_int<true>(g, h, lane, m, P, gc, tot_g, tot_h, gscale, hscale, num_data, min_gain_shift, parent_output, zero, na, &splittable);
    apply(r, true);
  }
  if (two_way) {
    const DirBestInt fw = scan_direction_int<false>(g, h, lane, m, P, gc, tot_g, tot_h, gscale, hscale, num_data, min_gain_shift, parent_output, zero, na, &splittable);
    apply(fw, false);
  } else if (m.missing == 2) {
    out.default_left = 0;
  }
  *is_splittable = splittable;
  return out;
}

struct BlockBest { double gain; int32_t real; int32_t feature; };   // per k_scan block: its best candidate

struct ScanArgs {
  const FeatMeta* feat;
  const uint8_t* feature_used;      // by-tree mask or nullptr
  int32_t num_features;
  Params params;
  const Leaf* leaves;
  Ctl* ctl;
  long long* pool;
  int64_t slot_stride;
  const uint8_t* splittable;        // [slot][num_features] FeatureHistogram::is_splittable_ (read-only here)
  uint8_t* splittable_new;          // [2][num_features]: 0/1 = new flag of (smaller, larger), 2 = leave unchanged
  Cand* cand;                       // [2][num_features]: smaller, larger
  BlockBest* block_best;            // [2][scan_blocks]
  CommPeers peers;                  // row-shard: whose pools to sum, which feature slice is mine
};

constexpr int kScanWarps = 8;

__device__ __forceinline__ Cand cand_none() {
  Cand out;
  out.gain = -INFINITY; out.feature = -1; out.threshold = 0; out.default_left = 1;
  out.lsg = out.lsh = out.lout = out.rsg = out.rsh = out.rout = 0.0; out.left_count = out.right_count = 0; out.pad = 0;
  out.real = 0x7fffffff; out.owner = 0; out.ilg = 0; out.ilh = 0;
  return out;
}

// Single GPU / feature-shard: grid = (ceil(F/8), 2); blockIdx.y = 0 scans the smaller child, 1 the larger child
// (= parent - smaller).  One warp per (feature, child); the larger-child warp re-derives the smaller child's
// fixed slice itself, so the two warps of a feature exchange nothing.
// Row-shard: grid = (ceil(f_cnt/8), 1) over this rank's feature slice; one warp handles BOTH children, and the
// smaller child's slice is first REDUCED over all ranks by reading every peer's pool slot through NVLink
// (the reduce-scatter of DataParallelTreeLearner, data_parallel_tree_learner.cpp:283+, fused into the scan's
// load phase; int64 fixed point => the sum is exact and order-independent).  The global slice is written back
// into this rank's own pool so that later subtractions (parent - smaller) stay local.
template <bool ROWS, bool QUANT>
__global__ void __launch_bounds__(kScanWarps * 32, ROWS ? 1 : 2) k_scan(const __grid_constant__ ScanArgs a) {
  Ctl* c = a.ctl;
  if (!c->cur_valid || !c->do_find) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr bool rows = ROWS;
  const int f = (rows ? a.peers.f_lo : 0) + blockIdx.x * kScanWarps + warp;
  const int f_end = rows ? a.peers.f_lo + a.peers.f_cnt : a.num_features;
  const int F = a.num_features;
  const int smaller = c->smaller, larger = c->larger;
  __shared__ double s_gain[2][kScanWarps];
  __shared__ int s_real[2][kScanWarps], s_feat[2][kScanWarps];
  __shared__ int s_ok;

  if (rows) {
    // every peer's local histogram of this iteration must be complete before anyone sums it
    if (threadIdx.x < a.peers.world) {
      if (!wait_seq(&a.peers.block[a.peers.rank]->hist_seq[threadIdx.x], c->hist_seq)) c->error = 1;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_ok = c->error ? 0 : 1;
    __syncthreads();
    if (!s_ok) return;
  }

  const int w_lo = rows ? 0 : blockIdx.y, w_hi = rows ? 2 : blockIdx.y + 1;     // which children this warp handles
  const bool in_range = f < f_end;
  bool used = false;
  int inherit_flag0 = 2;
  FeatMeta m = {};
  long long ig[8], ih[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { ig[k] = 0; ih[k] = 0; }
  int64_t slice = 0;

  if (in_range) {
    const Leaf& LS = a.leaves[smaller];
    used = (a.feature_used == nullptr) || a.feature_used[f];
    if (used && larger >= 0 && !a.splittable[static_cast<int64_t>(a.leaves[larger].slot) * F + f]) {
      // parent was not splittable on this feature (serial_tree_learner.cpp:397-402): both children inherit it
      used = false; inherit_flag0 = 0;
    }
    if (used) {
      m = a.feat[f];
      slice = (static_cast<int64_t>(m.col) * kBinsPerColumn + m.lo) * 2;
      const int64_t soff = static_cast<int64_t>(LS.slot) * a.slot_stride + slice;
      long long* hs = a.pool + soff;
      // smaller child's slice (row-shard: summed over every rank's local histogram)
      if (rows) {
        for (int r = 0; r < a.peers.world; ++r) {
          const long long* hp = a.peers.pool[r] + soff;
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int e = lane * 8 + k;
            if (e < m.nslice) { const longlong2 v = __ldcv(reinterpret_cast<const longlong2*>(hp + 2 * e)); ig[k] += v.x; ih[k] += v.y; }
          }
        }
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int e = lane * 8 + k;
          if (e < m.nslice) { const longlong2 v = *reinterpret_cast<const longlong2*>(hs + 2 * e); ig[k] = v.x; ih[k] = v.y; }
        }
      }
      if (m.mfb > 0) {
        // Dataset::FixHistogram: entry[mfb] = leaf total - sum(other entries); the stored mfb entry is ignored,
        // so it does not matter whether the smaller-child warp has already written it back
        long long og = 0, oh = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { if (lane * 8 + k != m.mfb) { og += ig[k]; oh += ih[k]; } }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) { og += __shfl_xor_sync(0xffffffffu, og, d); oh += __shfl_xor_sync(0xffffffffu, oh, d); }
        const long long tg = (QUANT ? LS.isum_g : __double2ll_rn(LS.sum_g * c->g_scale)) - og;
        const long long th = (QUANT ? LS.isum_h : __double2ll_rn(LS.sum_h * c->h_scale)) - oh;
#pragma unroll
        for (int k = 0; k < 8; ++k) { if (lane * 8 + k == m.mfb) { ig[k] = tg; ih[k] = th; } }
      }
      if (w_lo == 0) {
        // keep the fixed (row-shard: global) slice: this leaf's slot is a future parent
        if (rows) {
#pragma unroll
          for (int k = 0; k < 8; ++k) { const int e = lane * 8 + k; if (e < m.nslice) *reinterpret_cast<longlong2*>(hs + 2 * e) = make_longlong2(ig[k], ih[k]); }
        } else if (m.mfb > 0) {
#pragma unroll
          for (int k = 0; k < 8; ++k) { if (lane * 8 + k == m.mfb) *reinterpret_cast<longlong2*>(hs + 2 * m.mfb) = make_longlong2(ig[k], ih[k]); }
        }
      }
    }
  }

  // one child at a time (no per-child arrays: keeps the kernel at 2 CTAs/SM)
#pragma unroll 1
  for (int which = w_lo; which < w_hi; ++which) {
    Cand out = cand_none();
    int new_flag = (which == 0) ? inherit_flag0 : 2;
    if (used && !(which == 1 && larger < 0)) {
      const GainCfg gc = make_gain_cfg(a.params);
      int splittable = 0;
      if (QUANT) {
        // integer histograms: the pool holds the raw sums of the discretized gradients (scale 1)
        long long qg[8], qh[8];
        long long tot_g, tot_h; double po; int cnt;
        if (which == 0) {
          const Leaf& LS = a.leaves[smaller];
#pragma unroll
          for (int k = 0; k < 8; ++k) { qg[k] = ig[k]; qh[k] = ih[k]; }
          tot_g = LS.isum_g; tot_h = LS.isum_h; cnt = LS.count;
          po = (c->num_leaves == 1)
              ? leaf_output(GainCfg{1, 1, 0, a.params.l1, a.params.l2, a.params.max_delta_step, a.params.path_smooth}, LS.sum_g, LS.sum_h, LS.count, 0.0)
              : LS.output;
        } else {
          const Leaf& LL = a.leaves[larger];
          long long* hl = a.pool + static_cast<int64_t>(LL.slot) * a.slot_stride + slice;
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int e = lane * 8 + k;
            if (e < m.nslice) {
              longlong2 v = *reinterpret_cast<const longlong2*>(hl + 2 * e);
              v.x -= ig[k]; v.y -= ih[k];
              *reinterpret_cast<longlong2*>(hl + 2 * e) = v;
              qg[k] = v.x; qh[k] = v.y;
            } else { qg[k] = 0; qh[k] = 0; }
          }
          tot_g = LL.isum_g; tot_h = LL.isum_h; cnt = LL.count; po = LL.output;
        }
        out = find_best_threshold_int(qg, qh, lane, f, m, a.params, gc, tot_g, tot_h, c->q_gscale, c->q_hscale, cnt, po, &splittable);
      } else {
      const double g_inv = c->g_inv, h_inv = c->h_inv;
      double g[8], h[8];
      double sum_g, sum_h, po; int cnt;
      if (which == 0) {
        const Leaf& LS = a.leaves[smaller];
#pragma unroll
        for (int k = 0; k < 8; ++k) { h[k] = static_cast<double>(ih[k]) * h_inv; g[k] = static_cast<double>(ig[k]) * g_inv; }
        sum_g = LS.sum_g; sum_h = LS.sum_h; cnt = LS.count;
        po = (c->num_leaves == 1)
            ? leaf_output(GainCfg{1, 1, 0, a.params.l1, a.params.l2, a.params.max_delta_step, a.params.path_smooth}, LS.sum_g, LS.sum_h, LS.count, 0.0)
            : LS.output;
      } else {
        // larger child = parent - smaller (exact), written in place into the parent's slot
        const Leaf& LL = a.leaves[larger];
        long long* hl = a.pool + static_cast<int64_t>(LL.slot) * a.slot_stride + slice;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int e = lane * 8 + k;
          if (e < m.nslice) {
            longlong2 v = *reinterpret_cast<const longlong2*>(hl + 2 * e);
            v.x -= ig[k]; v.y -= ih[k];
            *reinterpret_cast<longlong2*>(hl + 2 * e) = v;
            h[k] = static_cast<double>(v.y) * h_inv;
            g[k] = static_cast<double>(v.x) * g_inv;
          } else { g[k] = 0.0; h[k] = 0.0; }
        }
        sum_g = LL.sum_g; sum_h = LL.sum_h; cnt = LL.count; po = LL.output;
      }
      out = find_best_threshold(g, h, lane, f, m, a.params, gc, sum_g, sum_h, cnt, po, &splittable);
      }
      new_flag = splittable;
    }
    if (lane == 0) {
      if (in_range && !(which == 1 && larger < 0 && !rows)) {
        a.cand[which * F + f] = out;
        a.splittable_new[which * F + f] = static_cast<uint8_t>(new_flag);
      }
      // block-level arg-max input (gain, then smaller real feature index) so that k_select scans F/8 entries only
      s_gain[which][warp] = out.gain; s_real[which][warp] = out.feature < 0 ? 0x7fffffff : out.real; s_feat[which][warp] = out.feature;
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 && static_cast<int>(threadIdx.x) >= w_lo && static_cast<int>(threadIdx.x) < w_hi) {
    const int which = threadIdx.x;
    BlockBest bb; bb.gain = -INFINITY; bb.real = 0x7fffffff; bb.feature = -1;
    for (int w = 0; w < kScanWarps; ++w) {
      if (s_feat[which][w] < 0) continue;
      if (s_gain[which][w] > bb.gain || (s_gain[which][w] == bb.gain && s_real[which][w] < bb.real)) { bb.gain = s_gain[which][w]; bb.real = s_real[which][w]; bb.feature = s_feat[which][w]; }
    }
    a.block_best[which * gridDim.x + blockIdx.x] = bb;
  }
}

// ---------------------------------------------------------------------------------------------------
// k_select: per-leaf arg-max over features (SplitInfo::operator>, split_info.hpp:138-164), then the
// arg-max over leaves (array_args.h:45-60) and the snapshot of the split to apply next.
struct SelectArgs {
  const FeatMeta* feat;
  int32_t num_features;
  int32_t max_leaves;
  Leaf* leaves;
  Ctl* ctl;
  const Cand* cand;
  const BlockBest* block_best;  // [2][scan_blocks]
  int32_t scan_blocks;
  uint8_t* splittable;          // [slot][num_features]
  const uint8_t* splittable_new;  // [2][num_features] written by k_scan
  CommPeers peers;              // world == 1: no exchange
};

// payload written by a peer GPU: read it around L1 (the acquire on the sequence word orders it)
__device__ __forceinline__ Cand load_cand_sys(const Cand* p) {
  static_assert(sizeof(Cand) % 8 == 0, "Cand must be a multiple of 8 bytes");
  Cand out;
  const unsigned long long* s = reinterpret_cast<const unsigned long long*>(p);
  unsigned long long* d = reinterpret_cast<unsigned long long*>(&out);
#pragma unroll
  for (int i = 0; i < static_cast<int>(sizeof(Cand) / 8); ++i) d[i] = __ldcv(s + i);
  return out;
}

__device__ __forceinline__ bool cand_better(double ga, int fa_real, double gb, int fb_real) {
  if (ga != gb) return ga > gb;
  return fa_real < fb_real;
}

__global__ void __launch_bounds__(256) k_select(const __grid_constant__ SelectArgs a) {
  Ctl* c = a.ctl;
  if (!c->cur_valid) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int F = a.num_features;
  const int smaller = c->smaller, larger = c->larger, do_find = c->do_find;

  // (1) warps 0/1: per-leaf arg-max over the k_scan block winners (SplitInfo::operator>) -> leaves[].best
  //     warps 2..7: hand the children's is_splittable_ flags over from the staging array
  if (warp < 2) {
    const int which = warp;
    const int leaf = which == 0 ? smaller : larger;
    if (leaf >= 0) {
      double bg = -INFINITY; int br = 0x7fffffff, bi = -1;
      if (do_find) {
        for (int b = lane; b < a.scan_blocks; b += 32) {
          const BlockBest bb = a.block_best[which * a.scan_blocks + b];
          if (bb.feature >= 0 && cand_better(bb.gain, bb.real, bg, br)) { bg = bb.gain; br = bb.real; bi = bb.feature; }
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
          const double og = __shfl_xor_sync(0xffffffffu, bg, d);
          const int orl = __shfl_xor_sync(0xffffffffu, br, d), oi = __shfl_xor_sync(0xffffffffu, bi, d);
          if (oi >= 0 && cand_better(og, orl, bg, br)) { bg = og; br = orl; bi = oi; }
        }
      }
      if (lane == 0) {
        Leaf& L = a.leaves[leaf];
        if (bi >= 0) { L.best = a.cand[which * F + bi]; L.best.owner = a.peers.rank; }
        else { L.best.gain = -INFINITY; L.best.feature = -1; L.best.real = 0x7fffffff; L.best.owner = a.peers.rank; }
      }
    }
  } else if (do_find) {
    for (int which = 0; which < 2; ++which) {
      const int leaf = which == 0 ? smaller : larger;
      if (leaf < 0) continue;
      uint8_t* dst = a.splittable + static_cast<int64_t>(a.leaves[leaf].slot) * F;
      const bool rows = a.peers.world > 1 && a.peers.mode == 1;       // row-shard: only my feature slice was scanned
      const int f0 = rows ? a.peers.f_lo : 0, f1 = rows ? a.peers.f_lo + a.peers.f_cnt : F;
      for (int f = f0 + tid - 64; f < f1; f += 192) { const uint8_t v = a.splittable_new[which * F + f]; if (v != 2) dst[f] = v; }
    }
  }
  __syncthreads();

  // (2) feature-shard: exchange the two per-leaf winners with every peer over NVLink peer memory and keep
  // the global best (SyncUpGlobalBestSplit, reference src/treelearner/parallel_tree_learner.h:207-232).
  // Every rank applies the same deterministic reduction => identical decisions everywhere.
  if (a.peers.world > 1) {
    const int W = a.peers.world, me = a.peers.rank;
    const unsigned long long seq = c->xchg_seq + 1;
    const int par = static_cast<int>(seq & 1);
    if (tid < W) {
      CommBlock* dst = a.peers.block[tid];
      Cand* slot = &dst->mail[par][me][0];
      slot[0] = a.leaves[smaller].best;
      if (larger >= 0) slot[1] = a.leaves[larger].best;
      st_release_sys(&dst->mail_seq[par][me], seq);
    }
    __syncthreads();
    if (tid < W) {
      CommBlock* mine = a.peers.block[me];
      if (!wait_seq(&mine->mail_seq[par][tid], seq)) c->error = 1;
    }
    __syncthreads();
    // warps 0 / 1 reduce the smaller / larger leaf: lane r reads only the KEY of rank r's candidate (gain, feature, real
    // index), the warp agrees on the winning rank by shuffles (the comparator of the sequential scan; among equals the
    // lower rank), and one lane copies the winner's full record.  (Reading all W records one after the other in one thread
    // was a chain of W dependent L2 round trips: several microseconds per split at 8 GPUs.)
    if (warp < 2) {
      const int which = warp;
      const int leaf = which == 0 ? smaller : larger;
      if (leaf >= 0) {
        CommBlock* mine = a.peers.block[me];
        double g = -INFINITY; int real = 0x7fffffff, win = 0x7fffffff;
        if (lane < W) {
          const Cand* p = &mine->mail[par][lane][which];
          g = __ldcv(&p->gain);
          const int f = __ldcv(&p->feature);
          real = f < 0 ? 0x7fffffff : __ldcv(&p->real);
          win = lane;
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
          const double og = __shfl_xor_sync(0xffffffffu, g, d);
          const int orl = __shfl_xor_sync(0xffffffffu, real, d), ow = __shfl_xor_sync(0xffffffffu, win, d);
          if (ow != 0x7fffffff && (win == 0x7fffffff || cand_better(og, orl, g, real) || (!cand_better(g, real, og, orl) && ow < win))) { g = og; real = orl; win = ow; }
        }
        if (lane == 0) a.leaves[leaf].best = load_cand_sys(&mine->mail[par][win][which]);
      }
    }
    __syncthreads();
    if (tid == 0) { c->xchg_seq = seq; if (c->error) c->cur_valid = 0; }
    __syncthreads();
    if (c->error) return;
  }

  // (3) warp 0: arg-max over all leaf slots (array_args.h:45-60: first maximum in leaf order under
  //     operator>; ungrown leaves hold gain = -inf, feature = -1), stop rule, snapshot of the split to apply
  if (warp == 0) {
    double bg = -INFINITY; int br = 0x7fffffff, bi = 0x7fffffff;
    for (int i = lane; i < a.max_leaves; i += 32) {
      const Cand& cd = a.leaves[i].best;
      const double g = cd.gain; const int real = cd.feature < 0 ? 0x7fffffff : cd.real;
      if (bi == 0x7fffffff || cand_better(g, real, bg, br)) { bg = g; br = real; bi = i; }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
      const double og = __shfl_xor_sync(0xffffffffu, bg, d);
      const int orl = __shfl_xor_sync(0xffffffffu, br, d), oi = __shfl_xor_sync(0xffffffffu, bi, d);
      if (oi != 0x7fffffff && (bi == 0x7fffffff || cand_better(og, orl, bg, br) ||
                               (!cand_better(bg, br, og, orl) && oi < bi))) { bg = og; br = orl; bi = oi; }
    }
    if (lane == 0) {
      const int best_leaf = bi;
      const Leaf& L = a.leaves[best_leaf];
      // serial_tree_learner.cpp:232: stop when the best gain is <= 0; also when the tree is full
      if (L.best.gain <= 0.0 || L.best.feature < 0 || c->num_leaves >= a.max_leaves) {
        c->cur_valid = 0;
      } else {
        c->cur_leaf = best_leaf; c->cur_begin = L.begin; c->cur_count = L.lcount; c->cur_buf = L.buf;
        c->cur_feature = L.best.feature; c->cur_threshold = L.best.threshold; c->cur_default_left = L.best.default_left;
        c->cur_owner = a.peers.mode == 1 ? a.peers.rank : L.best.owner;   // row-shard: every rank holds every column
        if (a.peers.mode == 2) c->cur_meta = a.peers.gmeta[a.peers.feat_off[L.best.owner] + L.best.feature];   // replicated columns
        else if (c->cur_owner == a.peers.rank) c->cur_meta = a.feat[L.best.feature];   // only the owner holds the column
        c->part_blocks_done = 0;
        c->flag_seq += 1;          // sequence number of the flag push that applies this split
      }
    }
  }
}

}  // namespace b200
