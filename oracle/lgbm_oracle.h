/*
 * lgbm_oracle.h — CPU restatement (plain C, fp64, single thread) of LightGBM's serial tree-learner
 * hot path.  TEST INFRASTRUCTURE ONLY: used by tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg as the checker for the CUDA path.  Never linked into / called from the product
 * library (lightgbm_b200/).
 *
 * Parity status: PINNED against the compiled reference (oracle/_ref/lib_lightgbm.so, built by
 * oracle/Makefile.ref from /root/reference) — see tests/test_oracle_vs_reference.py and the golden
 * fixtures under tests/golden/ produced by tests/golden/make_golden.py.
 *
 * All file:line citations are relative to /root/reference.
 */
#ifndef LGBM_ORACLE_H_
#define LGBM_ORACLE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* MissingType — include/LightGBM/bin.h:28-32 */
enum { ORC_MISSING_NONE = 0, ORC_MISSING_ZERO = 1, ORC_MISSING_NAN = 2 };

/*
 * The layout contract (SURVEY.md §8 a15): a row-major uint8 matrix [num_data x num_columns] of
 * *stored group values* exactly as FeatureGroup::PushData writes them (feature_group.h:253-267):
 *   0                      -> every sub-feature of the column sits in its most-frequent bin
 *   feat_lo[f] + i         -> feature f has bin (i + offset_f), offset_f = (feat_mfb[f] == 0)
 * A feature's histogram slice has (num_bin - offset) entries (feature_histogram.hpp:1429-1433).
 */
typedef struct {
  int32_t num_data;
  int32_t num_columns;
  int32_t num_features;
  const int32_t* feat_column;      /* [F] group column holding feature f (Dataset::feature2group_) */
  const int32_t* feat_lo;          /* [F] bin_offsets_[sub_feature]            (feature_group.h:60-70) */
  const int32_t* feat_num_bin;     /* [F] BinMapper::num_bin()                                         */
  const int32_t* feat_mfb;         /* [F] BinMapper::GetMostFreqBin()                                  */
  const int32_t* feat_default_bin; /* [F] BinMapper::GetDefaultBin()                                   */
  const int32_t* feat_missing;     /* [F] BinMapper::missing_type()                                    */
  const int32_t* feat_real_index;  /* [F] Dataset::RealFeatureIndex(f) — the tie-break key             */
  const int32_t* feat_in_group;    /* [F] number of features in f's group (num_feature_==1 selects the
                                          USE_MIN_BIN=false Split overload, dense_bin.hpp:427-447)     */
} OrcLayout;

/* The Config fields the path reads (include/LightGBM/config.h, SURVEY.md §5 "Config / flags") */
typedef struct {
  int32_t num_leaves;
  int32_t max_depth;               /* <=0: unlimited */
  int32_t min_data_in_leaf;
  double  min_sum_hessian_in_leaf;
  double  lambda_l1;
  double  lambda_l2;
  double  min_gain_to_split;
  double  max_delta_step;
  double  path_smooth;
} OrcParams;

/* One SplitInfo (split_info.hpp:22-56) as chosen for split #i, plus which leaf it split. */
typedef struct {
  int32_t leaf;            /* leaf that was split; left child keeps this id, right child = i+1 */
  int32_t feature;         /* inner feature index                                              */
  int32_t threshold;       /* threshold in feature-local bin units                             */
  int32_t default_left;
  int32_t left_count;      /* true counts from the partition (serial_tree_learner.cpp:795-799) */
  int32_t right_count;
  double  gain;            /* best_gain - min_gain_shift                                        */
  double  left_sum_gradient, left_sum_hessian, left_output;
  double  right_sum_gradient, right_sum_hessian, right_output;
  double  second_gain;     /* NOT a reference field: the largest gain among the candidates NOT taken when this split was
                              chosen (other thresholds, other features, other leaves), minus the same min_gain_shift.
                              The parity tests accept a divergence of the CUDA path only where gain - second_gain is
                              below the stated tolerance (SURVEY.md 8d margin rule).  -inf when there was no runner-up;
                              not tracked (= -inf) on the quantized path, which must match exactly. */
} OrcSplit;

typedef struct {
  int32_t  num_leaves;        /* leaves actually grown                                   */
  OrcSplit* splits;           /* [params.num_leaves-1], caller allocated                 */
  double*  leaf_value;        /* [params.num_leaves]                                     */
  double*  leaf_weight;       /* [params.num_leaves] sum_hessian                         */
  int32_t* leaf_count;        /* [params.num_leaves]                                     */
  int32_t* leaf_depth;        /* [params.num_leaves]                                     */
  int32_t* leaf_begin;        /* [params.num_leaves] segment of `indices` (DataPartition)*/
  int32_t* indices;           /* [num_data] final partition, caller allocated            */
  double   root_sum_gradient, root_sum_hessian;
} OrcTree;

/* Histogram of one leaf: fp64 (grad,hess) interleaved, 256 slots per column, FixHistogram NOT applied.
 * (MultiValDenseBin::ConstructHistogramInner multi_val_dense_bin.hpp:58-102 / DenseBin dense_bin.hpp:98-141) */
void orc_construct_histogram(const OrcLayout* L, const uint8_t* bins, const int32_t* indices, int32_t n,
                             const float* grad, const float* hess, double* hist /* [C*256*2] */);

/* FixHistogram + FindBestThreshold for one feature on a column-layout histogram (dataset.cpp:1519-1537,
 * feature_histogram.hpp:165-175, :830-1057).  Returns 1 if is_splittable_. */
int orc_find_best_threshold(const OrcLayout* L, const OrcParams* P, int feature, double* hist, int do_fix,
                            double sum_gradient, double sum_hessian, int32_t num_data,
                            double parent_output, OrcSplit* out);

/* DataPartition::Split for one leaf (data_partition.hpp:101-120, dense_bin.hpp:314-394); stable.
 * Writes left rows then right rows back into indices[0..n); returns left count. */
int32_t orc_partition(const OrcLayout* L, const uint8_t* bins, int feature, int threshold, int default_left,
                      int32_t* indices, int32_t n);

/* SerialTreeLearner::Train (serial_tree_learner.cpp:182-248).  bag_indices==NULL -> all rows.
 * feature_used: [F] by-tree column sampling mask or NULL.  Returns 0 on success. */
int orc_train_tree(const OrcLayout* L, const uint8_t* bins, const float* grad, const float* hess,
                   const int32_t* bag_indices, int32_t bag_count, const uint8_t* feature_used,
                   const OrcParams* P, OrcTree* out);

/* ---- Quantized-gradient training (Config::use_quantized_grad; SURVEY.md §8 f-2) -------------------------------
 * GradientDiscretizer::DiscretizeGradients (gradient_discretizer.cpp:68-160) without stochastic rounding
 * (Config::stochastic_rounding = false; the stochastic branch draws from per-thread std::mt19937 streams whose
 * layout depends on OMP_NUM_THREADS and is therefore not a fixed function of the inputs).  Writes the int8 values
 * as floats (exact) so that the fp64 histogram code can be reused: integer sums are exact in fp64.
 * random_g / random_h: optional [num_data] values in [0,1) replacing the 0.5 rounding offset (the stochastic form,
 * :120-139, with random_value_pos already applied); NULL -> deterministic rounding. */
typedef struct {
  int32_t num_grad_quant_bins;     /* config.h:638 */
  int32_t is_constant_hessian;
  int32_t renew_leaf;              /* Config::quant_train_renew_leaf (config.h:645) */
  double  grad_scale, hess_scale;  /* outputs of orc_discretize */
} OrcQuant;

void orc_discretize(const float* grad, const float* hess, int32_t num_data, OrcQuant* Q,
                    const double* random_g, const double* random_h, float* qgrad, float* qhess);

/* FixHistogramInt + FindBestThresholdInt for one feature (feature_histogram.hpp:176-189, :209-228, :1059-1350).
 * `hist` holds exact integer sums (as fp64); int_sum_g / int_sum_h are the leaf's integer totals. */
int orc_find_best_threshold_int(const OrcLayout* L, const OrcParams* P, int feature, double* hist, int do_fix,
                                int64_t int_sum_g, int64_t int_sum_h, double grad_scale, double hess_scale,
                                int32_t num_data, double parent_output, OrcSplit* out,
                                int64_t* best_left_int_g, int64_t* best_left_int_h);

/* SerialTreeLearner::Train with use_quantized_grad (serial_tree_learner.cpp:182-248 and the quantized branches
 * :195-197, :241-244, :308-328, :857-905, :979-989).  grad/hess are the ORIGINAL gradients; Q->grad_scale /
 * hess_scale are filled in. */
int orc_train_tree_quant(const OrcLayout* L, const uint8_t* bins, const float* grad, const float* hess,
                         const int32_t* bag_indices, int32_t bag_count, const uint8_t* feature_used,
                         const OrcParams* P, OrcQuant* Q, const double* random_g, const double* random_h, OrcTree* out);

#ifdef __cplusplus
}
#endif
#endif  /* LGBM_ORACLE_H_ */
