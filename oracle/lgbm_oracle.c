/*
 * lgbm_oracle.c — see lgbm_oracle.h.  TEST INFRASTRUCTURE ONLY (the checker, never the product).
 * A single-threaded, fp64, row-order restatement of the reference CPU learner so that, when the
 * reference is run with num_threads=1 / deterministic=true, histograms, gains and the split
 * sequence agree bit for bit.  Citations are relative to /root/reference.
 */
#include "lgbm_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

/* meta.h:50,54 — both constants are *float* literals widened to double at each use. */
static const double K_EPS = (double)1e-15f;
#define K_MIN_SCORE (-INFINITY)

/* common.h:910 RoundInt, common.h Sign */
static inline int round_int(double x) { return (int)(x + 0.5); }
static inline double sign_of(double x) { return (double)((x > 0.0) - (x < 0.0)); }

/* feature_histogram.hpp:711-714 */
static inline double threshold_l1(double s, double l1) {
  double r = fabs(s) - l1;
  if (r < 0.0) r = 0.0;
  return sign_of(s) * r;
}

typedef struct {
  int use_l1, use_max_output, use_smoothing; /* template dispatch feature_histogram.hpp:272-300 */
  double l1, l2, max_delta_step, smoothing;
} GainCfg;

static GainCfg gain_cfg(const OrcParams* P) {
  GainCfg c;
  c.use_l1 = P->lambda_l1 > 0.0;
  c.use_max_output = P->max_delta_step > 0.0;
  c.use_smoothing = P->path_smooth > K_EPS;
  c.l1 = P->lambda_l1; c.l2 = P->lambda_l2; c.max_delta_step = P->max_delta_step; c.smoothing = P->path_smooth;
  return c;
}

/* feature_histogram.hpp:716-738 CalculateSplittedLeafOutput (no monotone constraints) */
static double leaf_output(const GainCfg* c, double sg, double sh, int32_t n, double parent_output) {
  double ret = c->use_l1 ? -threshold_l1(sg, c->l1) / (sh + c->l2) : -sg / (sh + c->l2);
  if (c->use_max_output) {
    if (c->max_delta_step > 0 && fabs(ret) > c->max_delta_step) ret = sign_of(ret) * c->max_delta_step;
  }
  if (c->use_smoothing) {
    ret = ret * (n / c->smoothing) / (n / c->smoothing + 1) + parent_output / (n / c->smoothing + 1);
  }
  return ret;
}

/* feature_histogram.hpp:817-828 GetLeafGainGivenOutput */
static double leaf_gain_given_output(const GainCfg* c, double sg, double sh, double out) {
  double g = c->use_l1 ? threshold_l1(sg, c->l1) : sg;
  return -(2.0 * g * out + (sh + c->l2) * out * out);
}

/* feature_histogram.hpp:799-815 GetLeafGain */
static double leaf_gain(const GainCfg* c, double sg, double sh, int32_t n, double parent_output) {
  if (!c->use_max_output && !c->use_smoothing) {
    double g = c->use_l1 ? threshold_l1(sg, c->l1) : sg;
    return (g * g) / (sh + c->l2);
  }
  return leaf_gain_given_output(c, sg, sh, leaf_output(c, sg, sh, n, parent_output));
}

/* ------------------------------------------------------------------------------------------------ */

void orc_construct_histogram(const OrcLayout* L, const uint8_t* bins, const int32_t* indices, int32_t n,
                             const float* grad, const float* hess, double* hist) {
  const int C = L->num_columns;
  memset(hist, 0, sizeof(double) * (size_t)C * 256 * 2);
  /* column-major loop order == the col-wise CPU path (dataset.cpp:1390-1440): for each group the rows
   * are visited in leaf order and added in fp64 (dense_bin.hpp:109-137). */
  /* columns are independent and every cell keeps its row order, so threading over columns (only worth it for the
   * benchmark-scale parity tests) cannot change a single bit of the result */
#pragma omp parallel for schedule(dynamic, 4) if ((int64_t)n * C > (1 << 24))
  for (int c = 0; c < C; ++c) {
    double* h = hist + (size_t)c * 512;
    for (int32_t i = 0; i < n; ++i) {
      const int32_t r = indices ? indices[i] : i;
      const uint32_t v = bins[(size_t)r * C + c];
      h[2 * v] += (double)grad[r];
      h[2 * v + 1] += (double)hess[r];
    }
  }
}

typedef struct { double gain; int threshold; int left_count; double slg, slh; int found; } DirBest;

/* feature_histogram.hpp:830-1057 FindBestThresholdSequentially, one direction.
 * `d` points at the feature's slice (entry t <-> bin t+offset). */
static void scan_one_direction(const double* d, int num_bin, int offset, int default_bin, const OrcParams* P,
                               const GainCfg* gc, double sum_gradient, double sum_hessian, int32_t num_data,
                               double min_gain_shift, double parent_output, int reverse, int skip_default,
                               int na_as_missing, int* is_splittable, OrcSplit* out, double* top2) {
  double best_slg = NAN, best_slh = NAN, best_gain = K_MIN_SCORE;
  int32_t best_left_count = 0;
  int best_threshold = num_bin;
  const double cnt_factor = num_data / sum_hessian;

  if (reverse) {
    double srg = 0.0, srh = K_EPS;
    int32_t right_count = 0;
    const int t_end = 1 - offset;
    for (int t = num_bin - 1 - offset - na_as_missing; t >= t_end; --t) {
      if (skip_default && (t + offset) == default_bin) continue;
      const double g = d[2 * t], h = d[2 * t + 1];
      srg += g; srh += h;
      right_count += round_int(h * cnt_factor);
      if (right_count < P->min_data_in_leaf || srh < P->min_sum_hessian_in_leaf) continue;
      const int32_t left_count = num_data - right_count;
      if (left_count < P->min_data_in_leaf) break;
      const double slh = sum_hessian - srh;
      if (slh < P->min_sum_hessian_in_leaf) break;
      const double slg = sum_gradient - srg;
      const double cur = leaf_gain(gc, slg, slh, left_count, parent_output) +
                         leaf_gain(gc, srg, srh, right_count, parent_output);
      if (cur <= min_gain_shift) continue;
      *is_splittable = 1;
      if (cur > top2[0]) { top2[1] = top2[0]; top2[0] = cur; } else if (cur > top2[1]) top2[1] = cur;   /* checker only */
      if (cur > best_gain) {
        best_left_count = left_count; best_slg = slg; best_slh = slh;
        best_threshold = t - 1 + offset; best_gain = cur;
      }
    }
  } else {
    double slg = 0.0, slh = K_EPS;
    int32_t left_count = 0;
    int t = 0;
    const int t_end = num_bin - 2 - offset;
    if (na_as_missing && offset == 1) {
      /* materialise the implicit bin 0 (feature_histogram.hpp:945-961) */
      slg = sum_gradient; slh = sum_hessian - K_EPS; left_count = num_data;
      for (int i = 0; i < num_bin - offset; ++i) {
        slg -= d[2 * i]; slh -= d[2 * i + 1];
        left_count -= round_int(d[2 * i + 1] * cnt_factor);
      }
      t = -1;
    }
    for (; t <= t_end; ++t) {
      if (skip_default && (t + offset) == default_bin) continue;
      if (t >= 0) {
        slg += d[2 * t]; slh += d[2 * t + 1];
        left_count += round_int(d[2 * t + 1] * cnt_factor);
      }
      if (left_count < P->min_data_in_leaf || slh < P->min_sum_hessian_in_leaf) continue;
      const int32_t right_count = num_data - left_count;
      if (right_count < P->min_data_in_leaf) break;
      const double srh = sum_hessian - slh;
      if (srh < P->min_sum_hessian_in_leaf) break;
      const double srg = sum_gradient - slg;
      const double cur = leaf_gain(gc, slg, slh, left_count, parent_output) +
                         leaf_gain(gc, srg, srh, right_count, parent_output);
      if (cur <= min_gain_shift) continue;
      *is_splittable = 1;
      if (cur > top2[0]) { top2[1] = top2[0]; top2[0] = cur; } else if (cur > top2[1]) top2[1] = cur;   /* checker only */
      if (cur > best_gain) {
        best_left_count = left_count; best_slg = slg; best_slh = slh;
        best_threshold = t + offset; best_gain = cur;
      }
    }
  }

  if (*is_splittable && best_gain > out->gain + min_gain_shift) {
    out->threshold = best_threshold;
    out->left_output = leaf_output(gc, best_slg, best_slh, best_left_count, parent_output);
    out->left_count = best_left_count;
    out->left_sum_gradient = best_slg;
    out->left_sum_hessian = best_slh - K_EPS;
    out->right_output = leaf_output(gc, sum_gradient - best_slg, sum_hessian - best_slh,
                                    num_data - best_left_count, parent_output);
    out->right_count = num_data - best_left_count;
    out->right_sum_gradient = sum_gradient - best_slg;
    out->right_sum_hessian = sum_hessian - best_slh - K_EPS;
    out->gain = best_gain - min_gain_shift;
    out->default_left = reverse;
  }
}

int orc_find_best_threshold(const OrcLayout* L, const OrcParams* P, int f, double* hist, int do_fix,
                            double sum_gradient, double sum_hessian_in, int32_t num_data,
                            double parent_output, OrcSplit* out) {
  const int num_bin = L->feat_num_bin[f], mfb = L->feat_mfb[f];
  const int offset = (mfb == 0) ? 1 : 0;
  const int missing = L->feat_missing[f], default_bin = L->feat_default_bin[f];
  double* d = hist + ((size_t)L->feat_column[f] * 256 + L->feat_lo[f]) * 2;
  const GainCfg gc = gain_cfg(P);

  /* Dataset::FixHistogram (dataset.cpp:1519-1537): the never-stored most-frequent bin */
  if (do_fix && mfb > 0) {
    d[2 * mfb] = sum_gradient; d[2 * mfb + 1] = sum_hessian_in;
    for (int i = 0; i < num_bin; ++i) {
      if (i != mfb) { d[2 * mfb] -= d[2 * i]; d[2 * mfb + 1] -= d[2 * i + 1]; }
    }
  }

  /* FeatureHistogram::FindBestThreshold (feature_histogram.hpp:165-175) */
  out->default_left = 1;
  out->gain = K_MIN_SCORE;
  out->feature = f;
  const double sum_hessian = sum_hessian_in + 2 * K_EPS;
  /* BeforeNumerical (:177-196) */
  int is_splittable = 0;
  const double min_gain_shift = leaf_gain(&gc, sum_gradient, sum_hessian, num_data, parent_output) + P->min_gain_to_split;
  double top2[2] = {K_MIN_SCORE, K_MIN_SCORE};   /* the two largest candidate gains of this feature (parity checker's margin rule) */

  /* direction dispatch FuncForNumricalL3 (:396-441) */
  if (num_bin > 2 && missing != ORC_MISSING_NONE) {
    if (missing == ORC_MISSING_ZERO) {
      scan_one_direction(d, num_bin, offset, default_bin, P, &gc, sum_gradient, sum_hessian, num_data, min_gain_shift, parent_output, 1, 1, 0, &is_splittable, out, top2);
      scan_one_direction(d, num_bin, offset, default_bin, P, &gc, sum_gradient, sum_hessian, num_data, min_gain_shift, parent_output, 0, 1, 0, &is_splittable, out, top2);
    } else {
      scan_one_direction(d, num_bin, offset, default_bin, P, &gc, sum_gradient, sum_hessian, num_data, min_gain_shift, parent_output, 1, 0, 1, &is_splittable, out, top2);
      scan_one_direction(d, num_bin, offset, default_bin, P, &gc, sum_gradient, sum_hessian, num_data, min_gain_shift, parent_output, 0, 0, 1, &is_splittable, out, top2);
    }
  } else {
    scan_one_direction(d, num_bin, offset, default_bin, P, &gc, sum_gradient, sum_hessian, num_data, min_gain_shift, parent_output, 1, 0, 0, &is_splittable, out, top2);
    if (missing == ORC_MISSING_NAN) out->default_left = 0;
  }
  out->second_gain = top2[1] > K_MIN_SCORE ? top2[1] - min_gain_shift : K_MIN_SCORE;
  return is_splittable;
}

/* ---- quantized-gradient path -------------------------------------------------------------------- */

/* GradientDiscretizer::DiscretizeGradients (gradient_discretizer.cpp:68-160).  static_cast<int8_t>(double)
 * truncates toward zero. */
void orc_discretize(const float* grad, const float* hess, int32_t n, OrcQuant* Q,
                    const double* random_g, const double* random_h, float* qgrad, float* qhess) {
  double max_g = fabs((double)grad[0]), max_h = fabs((double)hess[0]);
  for (int32_t i = 0; i < n; ++i) {
    const double ag = fabs((double)grad[i]), ah = fabs((double)hess[i]);
    if (ag > max_g) max_g = ag;
    if (ah > max_h) max_h = ah;
  }
  Q->grad_scale = max_g / (double)(Q->num_grad_quant_bins / 2);
  Q->hess_scale = Q->is_constant_hessian ? max_h : max_h / (double)Q->num_grad_quant_bins;
  /* all-zero gradients: the reference would divide by zero here; both this restatement and the CUDA path map the
   * degenerate case to all-zero integers */
  const double inv_g = Q->grad_scale > 0.0 ? 1.0f / Q->grad_scale : 0.0, inv_h = Q->hess_scale > 0.0 ? 1.0f / Q->hess_scale : 0.0;
  for (int32_t i = 0; i < n; ++i) {
    const double g = grad[i];
    const double rg = random_g ? random_g[i] : 0.5;
    qgrad[i] = (float)(g >= 0.0f ? (int8_t)(g * inv_g + rg) : (int8_t)(g * inv_g - rg));
    if (Q->is_constant_hessian) qhess[i] = 1.0f;
    else qhess[i] = (float)(int8_t)((double)hess[i] * inv_h + (random_h ? random_h[i] : 0.5));
  }
}

typedef struct { double gain; int threshold; int64_t ilg, ilh; } IntBest;

/* feature_histogram.hpp:1059-1350 FindBestThresholdSequentiallyInt, one direction.  The reference packs
 * (gradient << bits | hessian) into one integer and picks 16/32-bit accumulators per leaf; with no overflow
 * (which its bit-width rule guarantees) that is exact integer arithmetic on the two sums, restated here with
 * separate int64 values. */
static void scan_one_direction_int(const double* d, int num_bin, int offset, int default_bin, const OrcParams* P,
                                   const GainCfg* gc, int64_t tot_g, int64_t tot_h, double grad_scale, double hess_scale,
                                   int32_t num_data, double min_gain_shift, double parent_output, int reverse,
                                   int skip_default, int na_as_missing, int* is_splittable, OrcSplit* out,
                                   int64_t* out_ilg, int64_t* out_ilh) {
  double best_gain = K_MIN_SCORE;
  int64_t best_ilg = 0, best_ilh = 0;
  int best_threshold = num_bin;
  const double cnt_factor = (double)num_data / (double)(uint32_t)tot_h;

  if (reverse) {
    int64_t rg = 0, rh = 0;
    const int t_end = 1 - offset;
    for (int t = num_bin - 1 - offset - na_as_missing; t >= t_end; --t) {
      if (skip_default && (t + offset) == default_bin) continue;
      rg += (int64_t)d[2 * t]; rh += (int64_t)d[2 * t + 1];
      const int32_t right_count = round_int((double)(uint32_t)rh * cnt_factor);
      const double srh = (double)(uint32_t)rh * hess_scale;
      if (right_count < P->min_data_in_leaf || srh < P->min_sum_hessian_in_leaf) continue;
      const int32_t left_count = num_data - right_count;
      if (left_count < P->min_data_in_leaf) break;
      const int64_t lg = tot_g - rg, lh = tot_h - rh;
      const double slh = (double)(uint32_t)lh * hess_scale;
      if (slh < P->min_sum_hessian_in_leaf) break;
      const double srg = (double)rg * grad_scale, slg = (double)lg * grad_scale;
      const double cur = leaf_gain(gc, slg, slh + K_EPS, left_count, parent_output) +
                         leaf_gain(gc, srg, srh + K_EPS, right_count, parent_output);
      if (cur <= min_gain_shift) continue;
      *is_splittable = 1;
      if (cur > best_gain) { best_ilg = lg; best_ilh = lh; best_threshold = t - 1 + offset; best_gain = cur; }
    }
  } else {
    int64_t lg = 0, lh = 0;
    int t = 0;
    const int t_end = num_bin - 2 - offset;
    if (na_as_missing && offset == 1) {
      lg = tot_g; lh = tot_h;
      for (int i = 0; i < num_bin - offset; ++i) { lg -= (int64_t)d[2 * i]; lh -= (int64_t)d[2 * i + 1]; }
      t = -1;
    }
    for (; t <= t_end; ++t) {
      if (skip_default && (t + offset) == default_bin) continue;
      if (t >= 0) { lg += (int64_t)d[2 * t]; lh += (int64_t)d[2 * t + 1]; }
      const int32_t left_count = round_int((double)(uint32_t)lh * cnt_factor);
      const double slh = (double)(uint32_t)lh * hess_scale;
      if (left_count < P->min_data_in_leaf || slh < P->min_sum_hessian_in_leaf) continue;
      const int32_t right_count = num_data - left_count;
      if (right_count < P->min_data_in_leaf) break;
      const int64_t rg = tot_g - lg, rh = tot_h - lh;
      const double srh = (double)(uint32_t)rh * hess_scale;
      if (srh < P->min_sum_hessian_in_leaf) break;
      const double srg = (double)rg * grad_scale, slg = (double)lg * grad_scale;
      const double cur = leaf_gain(gc, slg, slh + K_EPS, left_count, parent_output) +
                         leaf_gain(gc, srg, srh + K_EPS, right_count, parent_output);
      if (cur <= min_gain_shift) continue;
      *is_splittable = 1;
      if (cur > best_gain) { best_ilg = lg; best_ilh = lh; best_threshold = t + offset; best_gain = cur; }
    }
  }

  if (*is_splittable && best_gain > out->gain + min_gain_shift) {
    /* feature_histogram.hpp:1303-1346 */
    const int64_t irg = tot_g - best_ilg, irh = tot_h - best_ilh;
    const double slg = (double)best_ilg * grad_scale, slh = (double)(uint32_t)best_ilh * hess_scale;
    const double srg = (double)irg * grad_scale, srh = (double)(uint32_t)irh * hess_scale;
    const int32_t lc = round_int((double)(uint32_t)best_ilh * cnt_factor);
    const int32_t rc = round_int((double)(uint32_t)irh * cnt_factor);
    out->threshold = best_threshold;
    out->left_output = leaf_output(gc, slg, slh, lc, parent_output);
    out->left_count = lc;
    out->left_sum_gradient = slg; out->left_sum_hessian = slh;
    out->right_output = leaf_output(gc, srg, srh, rc, parent_output);
    out->right_count = rc;
    out->right_sum_gradient = srg; out->right_sum_hessian = srh;
    out->gain = best_gain - min_gain_shift;
    out->default_left = reverse;
    *out_ilg = best_ilg; *out_ilh = best_ilh;
  }
}

int orc_find_best_threshold_int(const OrcLayout* L, const OrcParams* P, int f, double* hist, int do_fix,
                                int64_t tot_g, int64_t tot_h, double grad_scale, double hess_scale,
                                int32_t num_data, double parent_output, OrcSplit* out,
                                int64_t* out_ilg, int64_t* out_ilh) {
  const int num_bin = L->feat_num_bin[f], mfb = L->feat_mfb[f];
  const int offset = (mfb == 0) ? 1 : 0;
  const int missing = L->feat_missing[f], default_bin = L->feat_default_bin[f];
  double* d = hist + ((size_t)L->feat_column[f] * 256 + L->feat_lo[f]) * 2;
  const GainCfg gc = gain_cfg(P);

  /* Dataset::FixHistogramInt (dataset.cpp:1540-1576) */
  if (do_fix && mfb > 0) {
    double fg = (double)tot_g, fh = (double)tot_h;
    for (int i = 0; i < num_bin; ++i) {
      if (i != mfb) { fg -= d[2 * i]; fh -= d[2 * i + 1]; }
    }
    d[2 * mfb] = fg; d[2 * mfb + 1] = fh;
  }

  /* FindBestThresholdInt (:176-189) + BeforeNumericalInt (:209-228) */
  out->default_left = 1;
  out->gain = K_MIN_SCORE;
  out->feature = f;
  int is_splittable = 0;
  const double sum_gradient = (double)(int32_t)tot_g * grad_scale;
  const double sum_hessian = (double)(uint32_t)tot_h * hess_scale;
  const double min_gain_shift = leaf_gain(&gc, sum_gradient, sum_hessian, num_data, parent_output) + P->min_gain_to_split;

#define SCAN_INT(rev, skip, na) scan_one_direction_int(d, num_bin, offset, default_bin, P, &gc, tot_g, tot_h, grad_scale, hess_scale, \
    num_data, min_gain_shift, parent_output, rev, skip, na, &is_splittable, out, out_ilg, out_ilh)
  if (num_bin > 2 && missing != ORC_MISSING_NONE) {
    if (missing == ORC_MISSING_ZERO) { SCAN_INT(1, 1, 0); SCAN_INT(0, 1, 0); }
    else { SCAN_INT(1, 0, 1); SCAN_INT(0, 0, 1); }
  } else {
    SCAN_INT(1, 0, 0);
    if (missing == ORC_MISSING_NAN) out->default_left = 0;
  }
#undef SCAN_INT
  return is_splittable;
}

/* FeatureGroup::Split -> DenseBin::Split -> SplitInner (feature_group.h:398-425, dense_bin.hpp:314-447) */
int32_t orc_partition(const OrcLayout* L, const uint8_t* bins, int f, int threshold, int default_left,
                      int32_t* indices, int32_t n) {
  const int C = L->num_columns, col = L->feat_column[f];
  const uint32_t default_bin = (uint32_t)L->feat_default_bin[f], mfb = (uint32_t)L->feat_mfb[f];
  const int missing = L->feat_missing[f];
  const int single = L->feat_in_group[f] == 1;
  /* min_bin/max_bin: feature_group.h:405-406; the single-feature overload passes min_bin = 1 */
  const uint32_t lo = (uint32_t)L->feat_lo[f];
  const uint32_t min_bin = single ? 1u : lo;
  const uint32_t max_bin = lo + (uint32_t)(L->feat_num_bin[f] - (mfb == 0 ? 1 : 0)) - 1;
  const int use_min_bin = !single;
  int miss_zero = 0, miss_na = 0, mfb_zero = 0, mfb_na = 0;
  if (missing == ORC_MISSING_ZERO) { miss_zero = 1; mfb_zero = (default_bin == mfb); }
  else if (missing == ORC_MISSING_NAN) { miss_na = 1; mfb_na = (max_bin == mfb + min_bin && mfb > 0); }

  uint8_t th = (uint8_t)(threshold + min_bin);
  uint8_t t_zero_bin = (uint8_t)(min_bin + default_bin);
  if (mfb == 0) { --th; --t_zero_bin; }
  const uint8_t minb = (uint8_t)min_bin, maxb = (uint8_t)max_bin;

  int32_t* left = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
  int32_t* right = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
  int32_t nl = 0, nr = 0;
  const int default_to_left = (mfb <= (uint32_t)threshold);
  const int missing_to_left = (miss_zero || miss_na) ? default_left : 0;
#define PUSH(to_left, idx) do { if (to_left) left[nl++] = (idx); else right[nr++] = (idx); } while (0)
  if (min_bin < max_bin) {
    for (int32_t i = 0; i < n; ++i) {
      const int32_t idx = indices[i];
      const uint8_t bin = bins[(size_t)idx * C + col];
      if ((miss_zero && !mfb_zero && bin == t_zero_bin) || (miss_na && !mfb_na && bin == maxb)) {
        PUSH(missing_to_left, idx);
      } else if ((use_min_bin && (bin < minb || bin > maxb)) || (!use_min_bin && bin == 0)) {
        if ((miss_na && mfb_na) || (miss_zero && mfb_zero)) PUSH(missing_to_left, idx);
        else PUSH(default_to_left, idx);
      } else if (bin > th) {
        PUSH(0, idx);
      } else {
        PUSH(1, idx);
      }
    }
  } else {
    const int max_bin_to_left = (maxb <= th);
    for (int32_t i = 0; i < n; ++i) {
      const int32_t idx = indices[i];
      const uint8_t bin = bins[(size_t)idx * C + col];
      if (miss_zero && !mfb_zero && bin == t_zero_bin) {
        PUSH(missing_to_left, idx);
      } else if (bin != maxb) {
        if ((miss_na && mfb_na) || (miss_zero && mfb_zero)) PUSH(missing_to_left, idx);
        else PUSH(default_to_left, idx);
      } else {
        if (miss_na && !mfb_na) PUSH(missing_to_left, idx);
        else PUSH(max_bin_to_left, idx);
      }
    }
  }
#undef PUSH
  memcpy(indices, left, sizeof(int32_t) * (size_t)nl);
  memcpy(indices + nl, right, sizeof(int32_t) * (size_t)nr);
  free(left); free(right);
  return nl;
}

/* SplitInfo::operator> (split_info.hpp:138-164) with the real feature index as tie-break */
static int split_better(const OrcSplit* a, int a_real, const OrcSplit* b, int b_real) {
  if (a->gain != b->gain) return a->gain > b->gain;
  int fa = a->feature < 0 ? INT32_MAX : a_real, fb = b->feature < 0 ? INT32_MAX : b_real;
  return fa < fb;
}

/* Q == NULL: full-precision path.  Q != NULL: grad/hess hold the discretized values (exact small integers) and
 * true_grad/true_hess the original gradients (only read by quant_train_renew_leaf). */
static int train_impl(const OrcLayout* L, const uint8_t* bins, const float* grad, const float* hess,
                      const int32_t* bag_indices, int32_t bag_count, const uint8_t* feature_used,
                      const OrcParams* P, OrcTree* T, const OrcQuant* Q, const float* true_grad, const float* true_hess) {
  const int F = L->num_features, C = L->num_columns, NL = P->num_leaves;
  int64_t* leaf_ig = (int64_t*)calloc(NL, sizeof(int64_t));     /* LeafSplits::int_sum_gradients_and_hessians_ */
  int64_t* leaf_ih = (int64_t*)calloc(NL, sizeof(int64_t));
  int64_t* best_ilg = (int64_t*)calloc(NL, sizeof(int64_t));    /* SplitInfo::left_sum_gradient_and_hessian */
  int64_t* best_ilh = (int64_t*)calloc(NL, sizeof(int64_t));
  const size_t HS = (size_t)C * 512;
  const GainCfg gc_root = {1, 1, 0, P->lambda_l1, P->lambda_l2, P->max_delta_step, P->path_smooth};

  double* pool = (double*)calloc(HS * (size_t)NL, sizeof(double));   /* HistogramPool, unlimited cache */
  uint8_t* splittable = (uint8_t*)malloc((size_t)NL * F);             /* FeatureHistogram::is_splittable_ */
  OrcSplit* best = (OrcSplit*)malloc(sizeof(OrcSplit) * (size_t)NL); /* best_split_per_leaf_ */
  double* leaf_sg = (double*)calloc(NL, sizeof(double));
  double* leaf_sh = (double*)calloc(NL, sizeof(double));
  if (!pool || !splittable || !best || !leaf_sg || !leaf_sh) return -1;
  memset(splittable, 1, (size_t)NL * F);

  /* BeforeTrain (serial_tree_learner.cpp:291-341): DataPartition::Init + root sums */
  int32_t n_root;
  if (bag_indices) { n_root = bag_count; memcpy(T->indices, bag_indices, sizeof(int32_t) * (size_t)bag_count); }
  else { n_root = L->num_data; for (int32_t i = 0; i < n_root; ++i) T->indices[i] = i; }
  for (int i = 0; i < NL; ++i) { best[i].feature = -1; best[i].gain = K_MIN_SCORE; best[i].second_gain = K_MIN_SCORE; T->leaf_begin[i] = 0; T->leaf_count[i] = 0; T->leaf_depth[i] = 0; }
  T->leaf_count[0] = n_root;
  double sg = 0.0, sh = 0.0;
  if (!Q) {
    for (int32_t i = 0; i < n_root; ++i) { const int32_t r = T->indices[i]; sg += grad[r]; sh += hess[r]; }
  } else {
    /* LeafSplits::Init(int8 ...) (leaf_splits.hpp:117-140 / :170-195): fp64 sums of int*scale + the packed int sum */
    for (int32_t i = 0; i < n_root; ++i) {
      const int32_t r = T->indices[i];
      sg += (double)grad[r] * Q->grad_scale; sh += (double)hess[r] * Q->hess_scale;
      leaf_ig[0] += (int64_t)grad[r]; leaf_ih[0] += (int64_t)hess[r];
    }
  }
  leaf_sg[0] = sg; leaf_sh[0] = sh;
  T->root_sum_gradient = sg; T->root_sum_hessian = sh;
  /* root output (serial_tree_learner.cpp:207-211): <USE_MC,L1,MAX_OUTPUT,!SMOOTHING>, num_data_ */
  T->leaf_value[0] = leaf_output(&gc_root, sg, sh, L->num_data, 0.0);
  T->leaf_weight[0] = sh;
  T->num_leaves = 1;

  int left_leaf = 0, right_leaf = -1;
  for (int split = 0; split < NL - 1; ++split) {
    /* BeforeFindBestSplit (:343-387) */
    int do_find = 1;
    if (P->max_depth > 0 && T->leaf_depth[left_leaf] >= P->max_depth) do_find = 0;
    const int32_t n_left = T->leaf_count[left_leaf];
    const int32_t n_right = right_leaf >= 0 ? T->leaf_count[right_leaf] : 0;
    if (do_find && n_right < P->min_data_in_leaf * 2 && n_left < P->min_data_in_leaf * 2) do_find = 0;
    if (!do_find) {
      best[left_leaf].gain = K_MIN_SCORE;
      if (right_leaf >= 0) best[right_leaf].gain = K_MIN_SCORE;
    } else {
      int smaller, larger;
      if (right_leaf < 0) { smaller = left_leaf; larger = -1; }
      else if (n_left < n_right) { smaller = left_leaf; larger = right_leaf; }
      else { smaller = right_leaf; larger = left_leaf; }
      /* histogram slots: the parent's buffer (always slot `left_leaf`, the parent's id) becomes the
       * larger child's; the smaller child gets the other slot (HistogramPool::Move, :372-385). */
      double *h_small, *h_large = NULL;
      uint8_t *sp_small, *sp_large = NULL;
      if (larger >= 0) {
        if (smaller == left_leaf) {
          /* Move(left -> right): parent's data now lives in slot right_leaf */
          memcpy(pool + HS * (size_t)right_leaf, pool + HS * (size_t)left_leaf, HS * sizeof(double));
          memcpy(splittable + (size_t)right_leaf * F, splittable + (size_t)left_leaf * F, (size_t)F);
        }
        h_large = pool + HS * (size_t)larger; sp_large = splittable + (size_t)larger * F;
      }
      h_small = pool + HS * (size_t)smaller; sp_small = splittable + (size_t)smaller * F;

      /* FindBestSplits (:393-409): inherit parent's is_splittable */
      uint8_t* used = (uint8_t*)malloc((size_t)F);
      for (int f = 0; f < F; ++f) {
        used[f] = 0;
        if (feature_used && !feature_used[f]) continue;
        if (sp_large && !sp_large[f]) { sp_small[f] = 0; continue; }
        used[f] = 1;
      }
      /* ConstructHistograms (:411-478) smaller leaf only; larger by subtraction */
      orc_construct_histogram(L, bins, T->indices + T->leaf_begin[smaller], T->leaf_count[smaller], grad, hess, h_small);

      /* parent output (GetParentOutput :1012-1025) */
      double po_small, po_large = 0.0;
      if (T->num_leaves == 1) po_small = leaf_output(&gc_root, leaf_sg[smaller], leaf_sh[smaller], T->leaf_count[smaller], 0.0);
      else { po_small = T->leaf_value[smaller]; po_large = T->leaf_value[larger]; }

      OrcSplit bs, bl; bs.feature = -1; bs.gain = K_MIN_SCORE; bl = bs;
      int bs_real = 0, bl_real = 0;
      double bs2 = K_MIN_SCORE, bl2 = K_MIN_SCORE;   /* runner-up candidate gain per leaf (checker only) */
      for (int f = 0; f < F; ++f) {
        if (!used[f]) continue;
        OrcSplit s; memset(&s, 0, sizeof(s));
        int64_t ilg = 0, ilh = 0;
        if (!Q) sp_small[f] = (uint8_t)orc_find_best_threshold(L, P, f, h_small, 1, leaf_sg[smaller], leaf_sh[smaller], T->leaf_count[smaller], po_small, &s);
        else sp_small[f] = (uint8_t)orc_find_best_threshold_int(L, P, f, h_small, 1, leaf_ig[smaller], leaf_ih[smaller], Q->grad_scale, Q->hess_scale,
                                                              T->leaf_count[smaller], po_small, &s, &ilg, &ilh);
        s.leaf = smaller;
        if (Q) s.second_gain = K_MIN_SCORE;
        if (split_better(&s, L->feat_real_index[f], &bs, bs_real)) { if (bs.feature >= 0 && bs.gain > bs2) bs2 = bs.gain; if (s.second_gain > bs2) bs2 = s.second_gain; }
        else if (s.gain > bs2) bs2 = s.gain;
        if (split_better(&s, L->feat_real_index[f], &bs, bs_real)) { bs = s; bs_real = L->feat_real_index[f]; best_ilg[smaller] = ilg; best_ilh[smaller] = ilh; }
        if (larger < 0) continue;
        /* FeatureHistogram::Subtract (feature_histogram.hpp:96-145) on the feature's slice */
        {
          const int nent = L->feat_num_bin[f] - (L->feat_mfb[f] == 0 ? 1 : 0);
          const size_t o = ((size_t)L->feat_column[f] * 256 + L->feat_lo[f]) * 2;
          for (int i = 0; i < nent * 2; ++i) h_large[o + i] -= h_small[o + i];
        }
        OrcSplit l; memset(&l, 0, sizeof(l));
        /* FixHistogram is NOT re-run for the larger leaf when subtracting (:581-597): its mfb entry is
         * parent(fixed) - smaller(fixed). */
        if (!Q) sp_large[f] = (uint8_t)orc_find_best_threshold(L, P, f, h_large, 0, leaf_sg[larger], leaf_sh[larger], T->leaf_count[larger], po_large, &l);
        else sp_large[f] = (uint8_t)orc_find_best_threshold_int(L, P, f, h_large, 0, leaf_ig[larger], leaf_ih[larger], Q->grad_scale, Q->hess_scale,
                                                              T->leaf_count[larger], po_large, &l, &ilg, &ilh);
        l.leaf = larger;
        if (Q) l.second_gain = K_MIN_SCORE;
        if (split_better(&l, L->feat_real_index[f], &bl, bl_real)) { if (bl.feature >= 0 && bl.gain > bl2) bl2 = bl.gain; if (l.second_gain > bl2) bl2 = l.second_gain; }
        else if (l.gain > bl2) bl2 = l.gain;
        if (split_better(&l, L->feat_real_index[f], &bl, bl_real)) { bl = l; bl_real = L->feat_real_index[f]; best_ilg[larger] = ilg; best_ilh[larger] = ilh; }
      }
      free(used);
      bs.leaf = smaller; bs.second_gain = bs2; best[smaller] = bs;
      if (larger >= 0) { bl.leaf = larger; bl.second_gain = bl2; best[larger] = bl; }
    }

    /* ArgMax over best_split_per_leaf_ (array_args.h:45-60) — all num_leaves slots, operator> */
    int best_leaf = 0;
    for (int i = 1; i < NL; ++i) {
      const int ri = best[i].feature >= 0 ? L->feat_real_index[best[i].feature] : 0;
      const int rb = best[best_leaf].feature >= 0 ? L->feat_real_index[best[best_leaf].feature] : 0;
      if (split_better(&best[i], ri, &best[best_leaf], rb)) best_leaf = i;
    }
    OrcSplit* s = &best[best_leaf];
    if (s->gain <= 0.0) break;  /* serial_tree_learner.cpp:232 (gain <= 0 -> stop) */
    /* checker only: the best candidate NOT taken at this step = max(runner-up inside the chosen leaf, other leaves' bests) */
    for (int i = 0; i < NL; ++i) if (i != best_leaf && best[i].feature >= 0 && best[i].gain > s->second_gain) s->second_gain = best[i].gain;

    /* SplitInner (:769-925) */
    const int next_leaf = T->num_leaves;
    const int32_t begin = T->leaf_begin[best_leaf], cnt = T->leaf_count[best_leaf];
    const int32_t nl = orc_partition(L, bins, s->feature, s->threshold, s->default_left, T->indices + begin, cnt);
    T->leaf_count[best_leaf] = nl;
    T->leaf_begin[next_leaf] = begin + nl;
    T->leaf_count[next_leaf] = cnt - nl;
    s->left_count = nl; s->right_count = cnt - nl;
    s->leaf = best_leaf;
    T->splits[split] = *s;
    /* Tree::Split (tree.h:543-585) */
    T->leaf_value[best_leaf] = isnan(s->left_output) ? 0.0 : s->left_output;
    T->leaf_weight[best_leaf] = s->left_sum_hessian;
    T->leaf_value[next_leaf] = isnan(s->right_output) ? 0.0 : s->right_output;
    T->leaf_weight[next_leaf] = s->right_sum_hessian;
    T->leaf_depth[next_leaf] = T->leaf_depth[best_leaf] + 1;
    T->leaf_depth[best_leaf] += 1;
    T->num_leaves += 1;
    /* children sums come from the SplitInfo (:857-878) */
    leaf_sg[best_leaf] = s->left_sum_gradient; leaf_sh[best_leaf] = s->left_sum_hessian;
    leaf_sg[next_leaf] = s->right_sum_gradient; leaf_sh[next_leaf] = s->right_sum_hessian;
    if (Q) {
      /* SplitInfo::{left,right}_sum_gradient_and_hessian -> LeafSplits::Init (serial_tree_learner.cpp:880-905) */
      const int64_t pg = leaf_ig[best_leaf], ph = leaf_ih[best_leaf];
      leaf_ig[best_leaf] = best_ilg[best_leaf]; leaf_ih[best_leaf] = best_ilh[best_leaf];
      leaf_ig[next_leaf] = pg - best_ilg[best_leaf]; leaf_ih[next_leaf] = ph - best_ilh[best_leaf];
    }
    left_leaf = best_leaf; right_leaf = next_leaf;
  }

  if (Q && Q->renew_leaf) {
    /* GradientDiscretizer::RenewIntGradTreeOutput (gradient_discretizer.cpp:236-259, serial_tree_learner.cpp:241-244):
     * leaf outputs from the ORIGINAL gradients, <USE_L1, USE_MAX_OUTPUT, !USE_SMOOTHING>, parent_output 0 */
    for (int leaf = 0; leaf < T->num_leaves; ++leaf) {
      double tg = 0.0, th = 0.0;
      const int32_t* idx = T->indices + T->leaf_begin[leaf];
      for (int32_t i = 0; i < T->leaf_count[leaf]; ++i) { tg += true_grad[idx[i]]; th += true_hess[idx[i]]; }
      T->leaf_value[leaf] = leaf_output(&gc_root, tg, th, T->leaf_count[leaf], 0.0);
    }
  }

  free(pool); free(splittable); free(best); free(leaf_sg); free(leaf_sh);
  free(leaf_ig); free(leaf_ih); free(best_ilg); free(best_ilh);
  return 0;
}

int orc_train_tree(const OrcLayout* L, const uint8_t* bins, const float* grad, const float* hess,
                   const int32_t* bag_indices, int32_t bag_count, const uint8_t* feature_used,
                   const OrcParams* P, OrcTree* T) {
  return train_impl(L, bins, grad, hess, bag_indices, bag_count, feature_used, P, T, NULL, NULL, NULL);
}

int orc_train_tree_quant(const OrcLayout* L, const uint8_t* bins, const float* grad, const float* hess,
                         const int32_t* bag_indices, int32_t bag_count, const uint8_t* feature_used,
                         const OrcParams* P, OrcQuant* Q, const double* random_g, const double* random_h, OrcTree* T) {
  float* qg = (float*)malloc(sizeof(float) * (size_t)L->num_data);
  float* qh = (float*)malloc(sizeof(float) * (size_t)L->num_data);
  if (!qg || !qh) return -1;
  orc_discretize(grad, hess, L->num_data, Q, random_g, random_h, qg, qh);
  const int rc = train_impl(L, bins, qg, qh, bag_indices, bag_count, feature_used, P, T, Q, grad, hess);
  free(qg); free(qh);
  return rc;
}
