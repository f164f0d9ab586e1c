/*
 * theia_matcher_b200.h -- C-ABI of the secondary path (SURVEY.md section 8, row a16): batched brute-force descriptor
 * matching behind theia::BruteForceFeatureMatcher (src/theia/matching/brute_force_feature_matcher.cc:49-117).
 * The per-pair hook MatchImagePair (feature_matcher.h:110-113) is too fine for a GPU; a maintainer overrides the
 * virtual FeatureMatcher::MatchImages (feature_matcher.h:97) to hand ALL image pairs to tbm_match_all and stores the
 * returned matches with FeaturesAndMatchesDatabase::PutImagePairMatch (INTEGRATION.md section 5).
 * Semantics are MatchImagePair's, per pair: squared float L2 (distance.h:52-56), best of image 2 for every descriptor of
 * image 1 (ties: lower index), kept if !use_lowes_ratio || best < ratio^2 * second (:78-81, double arithmetic on
 * float distances), early "not enough matches" exits (:84-86, :116), symmetric filtering through IntersectMatches
 * (feature_matcher_utils.cc:48-71).  128-dimensional descriptors (SIFT): a TF32 wgmma distance GEMM with a fused candidate-selection
 * epilogue selects candidates, an exact float pass (the reference's summation order) decides -- theiasfm_b200/csrc/tbm_matcher_tc.cuh;
 * other dimensions / TBM_PATH=exact: the round-1 CUDA-core kernel (bit-exact float summation order throughout).
 */
#ifndef THEIA_MATCHER_B200_H_
#define THEIA_MATCHER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* IndexedFeatureMatch, indexed_feature_match.h:40-52 */
typedef struct tbm_match { int32_t feature1_ind, feature2_ind; float distance; } tbm_match;

/* the FeatureMatcherOptions fields MatchImagePair reads (feature_matcher_options.h:45-71), same defaults */
typedef struct tbm_options {
  int32_t keep_only_symmetric_matches; /* 1 */
  int32_t use_lowes_ratio;             /* 1 */
  float lowes_ratio;                   /* 0.8f */
  int32_t min_num_feature_matches;     /* 30 */
} tbm_options;

void tbm_options_init(tbm_options* o);

/*
 * descriptors: [img_off[n_img]][dim] float (host), image i owns rows [img_off[i], img_off[i+1]).
 * pairs: [n_pairs][2] image indices.  For pair p the matches are written to matches[match_off[p] .. match_off[p+1])
 * (ascending feature1_ind); pair_ok[p] = MatchImagePair's return value (0 => the pair is dropped, its matches are the
 * ones found before the early exit, as in the reference).  Returns 0, or a negative code (-3 CUDA, -5 no device,
 * -1 bad argument / capacity too small: then match_off[n_pairs] holds the required capacity).
 */
int tbm_match_all(int device, const float* descriptors, const int64_t* img_off, int32_t n_img, int32_t dim,
                  const int32_t* pairs, int64_t n_pairs, const tbm_options* options, tbm_match* matches,
                  int64_t matches_capacity, int64_t* match_off /*[n_pairs+1]*/, uint8_t* pair_ok /*[n_pairs]*/);

/* Host restatement of the per-pair decisions (ratio test, early exits, intersection) that tbm_match_all takes on the device
 * (theiasfm_b200/csrc/tbm_decide.cuh: one CTA per pair, only the kept matches are copied back): exposed so that the CPU test
 * suite can pin the logic against the oracle without a GPU.  best_j / best_d / second_d: forward [n1] and
 * reverse [n2] results; second_valid = 0 when the other image has a single descriptor.  Returns MatchImagePair's bool. */
int tbm_debug_postprocess(const int32_t* f_best_j, const float* f_best_d, const float* f_second_d, int32_t n1, int f_second_valid,
                          const int32_t* r_best_j, const float* r_best_d, const float* r_second_d, int32_t n2, int r_second_valid,
                          const tbm_options* options, tbm_match* matches /* capacity n1 */, int32_t* n_matches);

/* Device times (CUDA events, ms) of the last tbm_match_all on the tensor-core path: {candidate GEMM kernel (wgmma), exact
 * re-evaluation kernel, host-to-device copy of the descriptors}; out4[3] = number of queries whose candidate list overflowed
 * and were scanned exhaustively by the exact pass.  All zero after a call that took the CUDA-core path. */
void tbm_debug_last_timing(double* out4);

/* Test hook: the exact re-evaluation kernel of the tensor-core path alone, on caller-made candidate lists (tests): descriptors
 * [n_rows][128]; query i = row q_row[i] against rows [b_row0[i], b_row0[i] + b_rows[i]); cand [n_q][16] global row indices
 * (-1 = empty slot; cand[i][0] == -2 or cand[i][8] == -2: scan every candidate of query i). */
int tbm_debug_exact_top2(int device, const float* descriptors, int64_t n_rows, const int32_t* q_row, const int32_t* b_row0,
                         const int32_t* b_rows, const int32_t* cand, int64_t n_q, int32_t* best_j, float* best_d, float* second_d);

/* Test hook: the nearest-neighbour stage of tbm_match_all alone (same inputs and path: the tensor-core path for dim 128 unless
 * TBM_PATH=exact), i.e. the per-query results the decision stage consumes.  For every pair, in pair order: its n1 forward queries,
 * then, when symmetric != 0, its n2 reverse queries.  best_j = nearest candidate (-1: the other image is empty), best_d / second_d =
 * exact float distances of the nearest and second-nearest (0 when missing); exhaustive[q] = 1 when the tensor-core candidate pass
 * handed query q to the exhaustive exact scan (always 0 on the CUDA-core path).  Returns 0 or a tbm_match_all error code. */
int tbm_debug_nn2(int device, const float* descriptors, const int64_t* img_off, int32_t n_img, int32_t dim, const int32_t* pairs,
                  int64_t n_pairs, int symmetric, int32_t* best_j, float* best_d, float* second_d, uint8_t* exhaustive);

#ifdef __cplusplus
}
#endif
#endif
