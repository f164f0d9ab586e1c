/*
 * theia_ba_b200.h -- C-ABI of the H100-native bundle-adjustment engine.
 *
 * This is the single drop-in boundary behind TheiaSfM's
 *   BundleAdjustReconstruction / BundleAdjustPartialReconstruction
 *     (src/theia/sfm/bundle_adjustment/bundle_adjustment.h:136-143,
 *      bundle_adjustment.cc:47-80)
 *   BundleAdjuster::{BundleAdjuster, AddView, AddTrack, Optimize}
 *     (src/theia/sfm/bundle_adjustment/bundle_adjuster.h:60-77,
 *      bundle_adjuster.cc:82-221)
 * The adapter (adapter/bundle_adjuster_b200.cc) performs what
 * bundle_adjuster.cc:102-180,223-371 performs against ceres::Problem --
 * deciding which parameter blocks / coordinates are constant -- and hands the
 * flattened problem to tba_solve(), which replaces the ceres::Solve() call at
 * bundle_adjuster.cc:205.  Everything is IEEE double; plain pointers and
 * sizes only (no torch / Eigen / ceres types).
 *
 * Parameter layouts follow the reference exactly:
 *   extrinsics [C_x C_y C_z  w_x w_y w_z]      camera.h:195-200
 *   PINHOLE    [f a s cx cy k1 k2]             pinhole_camera_model.h:86-94
 *   RADTAN     [f a s cx cy k1 k2 k3 t1 t2]    pinhole_radial_tangential_camera_model.h:91-102
 *   point      homogeneous [X Y Z h]           track.h:87
 */
#ifndef THEIA_BA_B200_H_
#define THEIA_BA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TBA_EXT_SIZE 6        /* Camera::kExtrinsicsSize, camera.h:200 */
#define TBA_INTR_STRIDE 10    /* max intrinsics size on this path (RADTAN) */
#define TBA_PT_SIZE 4         /* homogeneous point, track.h:87 */

/* CameraIntrinsicsModelType, camera_intrinsics_model_type.h:46-53 */
enum { TBA_MODEL_PINHOLE = 0, TBA_MODEL_PINHOLE_RADIAL_TANGENTIAL = 1, TBA_MODEL_FISHEYE = 2, TBA_MODEL_FOV = 3,
       TBA_MODEL_DIVISION_UNDISTORTION = 4 };
/* Number of intrinsic parameters of each model (NumParameters(): pinhole_camera_model.h:86-94 = 7,
 * pinhole_radial_tangential_camera_model.h:91-102 = 10, fisheye_camera_model.h:67-77 = 9, fov_camera_model.h:69-75 = 5,
 * division_undistortion_camera_model.h:76-82 = 5).  intr rows are always TBA_INTR_STRIDE wide; entries past the count
 * are ignored and returned unchanged. */
#define TBA_MODEL_NUM_PARAMETERS(model) \
  ((model) == 0 ? 7 : (model) == 1 ? 10 : (model) == 2 ? 9 : ((model) == 3 || (model) == 4) ? 5 : -1)

/* LossFunctionType, create_loss_function.h:51-58 */
enum { TBA_LOSS_TRIVIAL = 0, TBA_LOSS_HUBER = 1, TBA_LOSS_SOFTLONE = 2,
       TBA_LOSS_CAUCHY = 3, TBA_LOSS_ARCTAN = 4, TBA_LOSS_TUKEY = 5 };

/* OptimizeIntrinsicsType bitmask, bundle_adjustment.h:65-76 */
enum { TBA_INTR_NONE = 0x00, TBA_INTR_FOCAL_LENGTH = 0x01,
       TBA_INTR_ASPECT_RATIO = 0x02, TBA_INTR_SKEW = 0x04,
       TBA_INTR_PRINCIPAL_POINTS = 0x08, TBA_INTR_RADIAL_DISTORTION = 0x10,
       TBA_INTR_TANGENTIAL_DISTORTION = 0x20, TBA_INTR_ALL = 0x3f };

/* ceres::LinearSolverType / PreconditionerType numeric values (ceres/types.h,
 * pulled in by bundle_adjustment.h:38). */
enum { TBA_DENSE_NORMAL_CHOLESKY = 0, TBA_DENSE_QR = 1,
       TBA_SPARSE_NORMAL_CHOLESKY = 2, TBA_DENSE_SCHUR = 3,
       TBA_SPARSE_SCHUR = 4, TBA_ITERATIVE_SCHUR = 5, TBA_CGNR = 6 };
enum { TBA_PRECOND_IDENTITY = 0, TBA_PRECOND_JACOBI = 1,
       TBA_PRECOND_SCHUR_JACOBI = 2, TBA_PRECOND_CLUSTER_JACOBI = 3,
       TBA_PRECOND_CLUSTER_TRIDIAGONAL = 4 };

/* ext_const bits (what SetCameraPositionConstant / SetCameraOrientationConstant
 * / SetCameraExtrinsicsConstant at bundle_adjuster.cc:304-334 express). */
enum { TBA_EXT_POSITION_CONST = 1, TBA_EXT_ORIENTATION_CONST = 2,
       TBA_EXT_ALL_CONST = 3 };

/* Termination, mirroring ceres::TerminationType as used by
 * Summary::IsSolutionUsable() (bundle_adjuster.cc:218). */
enum { TBA_CONVERGENCE = 0, TBA_NO_CONVERGENCE = 1, TBA_FAILURE = 2 };

/* Return codes. */
enum { TBA_OK = 0, TBA_ERR_INVALID_ARGUMENT = -1, TBA_ERR_UNSUPPORTED = -2,
       TBA_ERR_CUDA = -3, TBA_ERR_NCCL = -4, TBA_ERR_NO_DEVICE = -5 };

/*
 * 1:1 POD mirror of theia::BundleAdjustmentOptions (bundle_adjustment.h:78-122;
 * same defaults via tba_options_init) followed by the ceres::Solver::Options
 * fields Theia leaves at Ceres' defaults but which define the trajectory.
 */
typedef struct tba_options {
  int32_t loss_function_type;          /* TRIVIAL */
  double  robust_loss_width;           /* 2.0 */
  int32_t linear_solver_type;          /* SPARSE_SCHUR; engine: ITERATIVE_SCHUR as such; every factorising type (0..4) = the same exact LM step, solved by PCG to the fp64 floor; CGNR refused */
  int32_t preconditioner_type;         /* SCHUR_JACOBI */
  int32_t visibility_clustering_type;  /* CANONICAL_VIEWS = 0 */
  int32_t verbose;                     /* 0 */
  int32_t constant_camera_orientation; /* 0 */
  int32_t constant_camera_position;    /* 0 */
  int32_t intrinsics_to_optimize;      /* FOCAL_LENGTH | RADIAL_DISTORTION */
  int32_t num_threads;                 /* 1 (host threads; unused on GPU) */
  int32_t max_num_iterations;          /* 100 */
  double  max_solver_time_in_seconds;  /* 3600 */
  int32_t use_inner_iterations;        /* 1 in Theia: coordinate descent over extrinsics / intrinsics / points after every LM step (DESIGN.md N4) */
  double  function_tolerance;          /* 1e-6 */
  double  gradient_tolerance;          /* 1e-10 */
  double  parameter_tolerance;         /* 1e-8 */
  double  max_trust_region_radius;     /* 1e12 */
  /* --- Ceres defaults not exposed by Theia --- */
  double  initial_trust_region_radius; /* 1e4 */
  double  min_trust_region_radius;     /* 1e-32 */
  double  min_relative_decrease;       /* 1e-3 */
  double  min_lm_diagonal;             /* 1e-6 */
  double  max_lm_diagonal;             /* 1e32 */
  double  eta;                         /* 1e-1 (CG q-tolerance) */
  int32_t min_linear_solver_iterations;/* 0 */
  int32_t max_linear_solver_iterations;/* 500 */
  int32_t jacobi_scaling;              /* 1 */
  int32_t max_num_consecutive_invalid_steps; /* 5 */
  int32_t cg_residual_reset_period;    /* 10 */
} tba_options;

/*
 * Flattened BA problem.  All arrays are caller-owned HOST memory; ext / intr /
 * pt are updated in place on return (variable coordinates only -- constant
 * coordinates come back bit-identical, like SubsetParameterization).
 */
typedef struct tba_problem {
  int32_t n_cam;
  double* ext;                    /* [n_cam * 6] in/out */
  const uint8_t* ext_const;       /* [n_cam] TBA_EXT_* bits */
  const int32_t* cam_group;       /* [n_cam] intrinsics group of each camera */
  int32_t n_group;
  const int32_t* group_model;     /* [n_group] TBA_MODEL_* */
  double* intr;                   /* [n_group * TBA_INTR_STRIDE] in/out */
  const uint32_t* group_const_mask; /* [n_group] bit j set => parameter j constant */
  int32_t n_pt;
  double* pt;                     /* [n_pt * 4] in/out */
  const uint8_t* pt_const;        /* [n_pt] nonzero => point block constant */
  int64_t n_obs;
  const int32_t* obs_cam;         /* [n_obs] */
  const int32_t* obs_pt;          /* [n_obs] */
  const double* obs_xy;           /* [n_obs * 2] Feature (feature.h:47) */
} tba_problem;

/* One row of the per-iteration table (the columns of Ceres'
 * PER_MINIMIZER_ITERATION log, bundle_adjuster.cc:63-64). */
typedef struct tba_iteration {
  int32_t iteration;
  int32_t step_is_valid;
  int32_t step_is_successful;
  int32_t linear_solver_iterations;
  double cost;
  double cost_change;
  double gradient_max_norm;
  double step_norm;
  double relative_decrease;
  double trust_region_radius;
  double iteration_time_in_seconds; /* device time of this iteration */
} tba_iteration;

/* theia::BundleAdjustmentSummary (bundle_adjustment.h:125-133) + detail. */
typedef struct tba_summary {
  int32_t success;
  double initial_cost;
  double final_cost;
  double setup_time_in_seconds;
  double solve_time_in_seconds;
  int32_t termination_type;
  int32_t num_iterations;            /* rows written to iterations[] */
  int32_t num_successful_steps;
  int32_t num_unsuccessful_steps;
  int32_t num_linear_solver_iterations;
  int64_t num_kernel_launches;       /* kernels launched by the engine */
  double h2d_bytes;
  double d2h_bytes;
  tba_iteration* iterations;         /* optional caller buffer */
  int32_t iterations_capacity;
  char message[256];
} tba_summary;

/* A context is NOT re-entrant: one solve at a time per context (Theia's estimators call full BA from a single
 * thread; bundle_adjuster.h's BundleAdjuster is not thread-safe either).  Different contexts may be used from
 * different threads concurrently. */
typedef struct tba_context tba_context;

/* Fill *o with theia::BundleAdjustmentOptions' defaults + Ceres' defaults. */
void tba_options_init(tba_options* o);

/* Number of visible CUDA devices (0 when none / driver missing). */
int tba_device_count(void);

/*
 * Persistent engine context for one GPU (streams, workspaces, NCCL comm).
 * rank/world_size/nccl_unique_id describe the one-process-per-GPU group the
 * context belongs to; world_size==1 needs no id.  nccl_unique_id is the 128
 * bytes of a ncclUniqueId obtained from tba_nccl_unique_id() on rank 0 and
 * broadcast by the host.
 */
int tba_create(int device, int rank, int world_size, const void* nccl_unique_id,
               tba_context** out);
void tba_destroy(tba_context* ctx);
int tba_nccl_unique_id(void* out_128_bytes);
const char* tba_last_error(tba_context* ctx);

/*
 * Replaces ceres::Solve (bundle_adjuster.cc:205).  Host buffers in, host
 * buffers out; H2D / D2H inside.  With world_size>1 every rank passes ITS
 * shard of points+observations (cameras/groups replicated); see
 * tba_shard_points().
 */
int tba_solve(tba_context* ctx, const tba_options* options,
              tba_problem* problem, tba_summary* summary);

/*
 * Single-process multi-GPU form of tba_solve for callers that, like Theia's estimators, run BA from one host
 * thread: shards points + observations over n_devices GPUs of the box (0 = all visible), one rank per device on
 * its own host thread, NCCL all-reduce of the camera-space sums.  Contexts are created once per process.
 */
int tba_solve_multi(const tba_options* options, tba_problem* problem, tba_summary* summary, int n_devices);

/*
 * Split-phase variant used by the benchmark and tests: upload+pack once,
 * iterate on device-resident data, download.
 */
int tba_upload(tba_context* ctx, const tba_options* options, const tba_problem* problem);
int tba_minimize(tba_context* ctx, tba_summary* summary);
int tba_download(tba_context* ctx, tba_problem* problem);

/*
 * N1 (SURVEY 8f): SetOutlierTracksToUnestimated (src/theia/sfm/set_outlier_tracks_to_unestimated.cc:62-136) evaluated on
 * the device-resident problem of this context (after tba_solve / tba_minimize), without a D2H -> hash-map -> reproject
 * round trip.  status[q] (q = caller point index): 0 keep, 1 bad reprojection (negative depth in a view, or mean squared
 * reprojection error > max_inlier_reprojection_error^2), 2 insufficient triangulation angle.  mean_sq_error (optional):
 * the per-track mean squared reprojection error of ComputeStatisticsForTrack
 * (select_good_tracks_for_bundle_adjustment.cc:79-108).  The return value of the reference = *bad + *insufficient.
 */
int tba_filter_tracks(tba_context* ctx, double max_inlier_reprojection_error, double min_triangulation_angle_degrees,
                      uint8_t* status, double* mean_sq_error, int32_t* num_bad_reprojections, int32_t* num_insufficient_angles);

/*
 * N3 (SURVEY 8f), batched micro-BA on the device-resident problem of this context (after tba_upload; read the points
 * back with tba_download).  Every camera and intrinsics block is held constant, whatever ext_const / group_const_mask
 * say; points with pt_const != 0 are skipped (status 255).
 *
 * tba_adjust_tracks = BundleAdjustTrack (src/theia/sfm/bundle_adjustment/bundle_adjustment.cc:96-107, DENSE_QR, no inner
 * iterations) for every non-constant point at once: status[q] = ceres termination (TBA_CONVERGENCE / NO_CONVERGENCE /
 * FAILURE; BundleAdjustmentSummary::success = status != TBA_FAILURE), initial_cost / final_cost optional [n_pt]
 * (-1 where no solve ran).  options: loss, tolerances, max_num_iterations, trust-region fields of tba_options.
 *
 * tba_estimate_tracks = TrackEstimator::EstimateTrack (src/theia/sfm/estimate_track.cc:199-264) for every non-constant
 * point at once, from the observations of the problem (the caller lists only estimated views, as
 * GetObservationsFromTrackViews does): viewing rays -> SufficientTriangulationAngle -> TriangulateMidpoint ->
 * BundleAdjustTrack (if bundle_adjustment) -> AcceptableReprojectionError.  The incoming point value is ignored.
 * status[q]: 0 estimated (the reference's "return true"), 1 fewer than 2 views or insufficient angle (num_bad_angles_),
 * 2 triangulation failed, 3 per-track BA failed, 4 unacceptable reprojection error (num_bad_reprojections_).
 * Like the reference, a track that fails at stage n keeps the point written by stage n-1.  counts[5] (optional) =
 * histogram of status 0..4.
 */
int tba_adjust_tracks(tba_context* ctx, const tba_options* options, uint8_t* status, double* initial_cost, double* final_cost,
                      int32_t* num_failed);
int tba_estimate_tracks(tba_context* ctx, const tba_options* ba_options, double max_acceptable_reprojection_error_pixels,
                        double min_triangulation_angle_degrees, int32_t bundle_adjustment, uint8_t* status, int32_t counts[5]);
enum { TBA_TRACK_ESTIMATED = 0, TBA_TRACK_BAD_ANGLE = 1, TBA_TRACK_TRIANGULATION_FAILED = 2, TBA_TRACK_BA_FAILED = 3,
       TBA_TRACK_BAD_REPROJECTION = 4, TBA_TRACK_SKIPPED = 255 };

/*
 * N3: BundleAdjustView (src/theia/sfm/bundle_adjustment/bundle_adjustment.cc:83-93, DENSE_QR, no inner iterations) for every
 * camera views[0..n_views) of the uploaded problem at once -- what LocalizeViewToReconstruction runs last for each newly
 * localized view (localize_view_to_reconstruction.cc:246-252).  Per view: one reprojection residual per observation of that
 * camera, every point constant, the free parameters are the camera's extrinsics and its intrinsics group with the coordinates
 * ext_const / group_const_mask of the upload leave free (at most 6 + 10).  options: loss and width, max_num_iterations,
 * tolerances and trust-region fields of tba_options; linear_solver_type and use_inner_iterations are ignored.  A view without
 * observations or without a free coordinate converges at iteration 0, parameters untouched, initial = final cost = its cost.
 * status[v]: TBA_CONVERGENCE / NO_CONVERGENCE / FAILURE (BundleAdjustmentSummary::success = status != TBA_FAILURE);
 * initial_cost / final_cost / iterations: optional, [n_views] (-1 costs where the initial evaluation failed).
 * Read the refined ext / intr back with tba_download; nothing else changes.
 * TBA_ERR_INVALID_ARGUMENT, with nothing changed: a view index out of range or listed twice, or two views that share an
 * intrinsics group with a free coordinate (one call per view would see the previous call's intrinsics -- adjust such views in
 * separate calls).  TBA_ERR_UNSUPPORTED on a context of a multi-rank group.
 */
int tba_adjust_views(tba_context* ctx, const tba_options* options, const int32_t* views, int32_t n_views, uint8_t* status,
                     double* initial_cost, double* final_cost, int32_t* iterations);

/*
 * N3: BundleAdjustTwoViews (src/theia/sfm/bundle_adjustment/bundle_adjust_two_views.cc:112-191) for MANY image pairs in one
 * call -- what TwoViewMatchGeometricVerification issues once per pair (two_view_match_geometric_verification.cc:268-296).
 * Per pair: camera 1 fixed, camera 2's extrinsics free, each camera's intrinsics constant or focal-length-only, every point
 * free, no robust loss, exact (DENSE_SCHUR) step, 200 iterations, Ceres' default tolerances -- all fixed by the reference
 * (.cc:54-69), so there is no options argument.  Pair p owns correspondences [pair_off[p], pair_off[p+1]).  The two cameras of
 * a pair have their own intrinsics rows.  Independent of any uploaded problem; ctx supplies device and stream.
 * termination[p]: TBA_CONVERGENCE / NO_CONVERGENCE / FAILURE (BundleAdjustmentSummary::success = termination != FAILURE,
 * .cc:185); initial_cost / final_cost / iterations: optional, [n_pairs].
 */
typedef struct tba_two_view_batch {
  int32_t n_pairs;
  const int64_t* pair_off;               /* [n_pairs + 1] */
  const double* ext1;                    /* [n_pairs * 6] camera 1 extrinsics (held constant) */
  double* ext2;                          /* [n_pairs * 6] in/out */
  double* intr1;                         /* [n_pairs * TBA_INTR_STRIDE] in/out (only the focal length can change) */
  double* intr2;                         /* [n_pairs * TBA_INTR_STRIDE] in/out */
  const int32_t* model1;                 /* [n_pairs] TBA_MODEL_* */
  const int32_t* model2;
  const uint8_t* constant_intrinsics1;   /* [n_pairs] TwoViewBundleAdjustmentOptions::constant_camera1_intrinsics */
  const uint8_t* constant_intrinsics2;
  const double* xy1;                     /* [n_corr * 2] FeatureCorrespondence::feature1 */
  const double* xy2;                     /* [n_corr * 2] feature2 */
  double* points;                        /* [n_corr * 4] in/out triangulated points */
  /* optional post-BA inlier test of BundleAdjustRelativePose (two_view_match_geometric_verification.cc:294-312): inlier[i] = both
   * cameras see point i at non-negative depth with squared reprojection error < final_max_reprojection_error_pixels^2 (:72-83).
   * inlier == NULL: skipped. */
  double final_max_reprojection_error_pixels;
  uint8_t* inlier;                       /* [n_corr] out, optional */
} tba_two_view_batch;
int tba_two_view_ba_batch(tba_context* ctx, tba_two_view_batch* batch, uint8_t* termination, double* initial_cost, double* final_cost,
                          int32_t* iterations);
/* The same over n_devices GPUs of the box (0 = all visible): pairs are independent units, so the batch is split into contiguous
 * ranges balanced by correspondence count and every range runs on its own device from its own host thread -- no collective.
 * Its contexts (one per device, no NCCL) are created once per process. */
int tba_two_view_ba_batch_multi(tba_two_view_batch* batch, int n_devices, uint8_t* termination, double* initial_cost, double* final_cost,
                                int32_t* iterations);

/* Re-load ext / intr / pt of an uploaded problem (same shape) without re-packing. */
int tba_reset_parameters(tba_context* ctx, const tba_problem* problem);
/* Change Solver::Options::max_num_iterations (bundle_adjustment.h:110) of an uploaded problem without re-packing. */
int tba_set_max_iterations(tba_context* ctx, int32_t max_num_iterations);

/* Per-kernel device timing (CUDA events on the engine stream) for the roofline report:
 * out[0..3] = {ms in the Schur matvec kernel, launches, ms in the linearise kernel, launches},
 * out[4..7] = {observation slots, observations, packed points, doubles stored per observation}. */
int tba_set_profiling(tba_context* ctx, int enable);
int tba_get_profile(tba_context* ctx, double* out8);
/* Per-stage breakdown of the same profiled run: out16[2k] = total ms, out16[2k+1] = launches, k over
 * {Schur matvec, linearise, extrinsics preconditioner blocks, intrinsics preconditioner blocks, reduced rhs,
 *  back-substitution, candidate cost, fused prepare (rhs + both preconditioner block families in one pass over J)}. */
int tba_get_profile_stages(tba_context* ctx, double* out16);

/* Contiguous point range [begin,end) owned by `rank` of `world_size`
 * (balanced by observation count given per-point counts). */
void tba_shard_points(const int32_t* pt_num_obs, int32_t n_pt, int world_size,
                      int rank, int32_t* begin, int32_t* end);

/*
 * Test / profiling hooks (kernel-level parity against oracle/): run single
 * stages on the uploaded problem and read back device vectors.
 */
enum { TBA_VEC_GRADIENT_CAM = 0,  /* [n_cam*6]            J^T r, unscaled      */
       TBA_VEC_GRADIENT_INTR = 1, /* [n_group*10]                               */
       TBA_VEC_GRADIENT_PT = 2,   /* [n_pt*4]                                   */
       TBA_VEC_COLNORM2_CAM = 3,  /* squared column norms of the unscaled J     */
       TBA_VEC_COLNORM2_INTR = 4,
       TBA_VEC_COLNORM2_PT = 5,
       TBA_VEC_RESIDUALS = 6,     /* [n_obs*2] (robustified), caller obs order  */
       TBA_VEC_SCHUR_RHS_CAM = 7, /* reduced rhs (Jacobi-scaled system)         */
       TBA_VEC_SCHUR_RHS_INTR = 8,
       TBA_VEC_PRECOND_CAM = 9,   /* [n_cam*36] inverse SCHUR_JACOBI blocks     */
       TBA_VEC_PRECOND_INTR = 10, /* [n_group*100]                              */
       TBA_VEC_STEP_CAM = 11,     /* last LM step (unscaled delta)              */
       TBA_VEC_STEP_INTR = 12,
       TBA_VEC_STEP_PT = 13 };
/* Host-only (no CUDA, no context): the observation packing tba_upload performs (DESIGN.md section 4), into caller
 * buffers of capacity cap_slots slots; sizes_out = {n_tiles, n_slots, n_packed_points, n_long_points, NI, imask}. */
int tba_debug_pack(const tba_problem* problem, int64_t cap_slots, int64_t* sizes_out, int32_t* slot_cam, int32_t* slot_pt,
                   int16_t* slot_run, uint8_t* slot_flags, double* xy, int64_t* slot_orig, int32_t* pk2caller,
                   int32_t* tile_pt_begin, int32_t* tile_nruns, uint8_t* tile_flags, double* mask);
int tba_debug_linearize(tba_context* ctx, double* cost);
/* One linearisation at the current parameters, returning the raw device buffers: J [n_slots/32][NJ][32], res [n_slots/32][2][32],
 * Hpp [n_pt][10], gp [n_pt][4] (packed points), lin [2 ncs + 3] = gradient | squared column norms | cost, fixed cost, failed
 * evaluations.  tile_kernel != 0: the tile-per-CTA kernel over every tile instead of the streaming kernel over the normal tiles.
 * sizes_out = {n_slots, NJ, n_pt, ncs}; with any output pointer NULL only the sizes are returned. */
int tba_debug_linearize_raw(tba_context* ctx, int tile_kernel, int64_t* sizes_out, double* J, double* res, double* Hpp,
                            double* gp, double* lin);
/* The intrinsics columns J_i of every observation slot as the passes over the stored linearisation see them (rebuilt from the
 * normalised image point in the compact layout, the stored rows otherwise), from the last linearisation:
 * Ji [n_slots/32][2 NI][32], in the order of the rows 14.. of J in the full layout.  sizes_out = {n_slots, NI}; with Ji NULL only
 * the sizes are returned. */
int tba_debug_intr_cols(tba_context* ctx, int64_t* sizes_out, double* Ji);
/* Launch geometry of the persistent warp-slice kernels over the normal tiles of the uploaded problem (no launch):
 * out[16] = {n_sm, n_slices, imask, has_ext_models, then {grid, warps per CTA, ring stages} of k_linearize_stream,
 * k_prepare_stream, k_schur_stream MODE 0 (matvec) and k_schur_stream MODE 1 / 2 (reduced rhs, back-substitution)}.
 * Warp gw of GW = grid * warps owns the slices [n_slices*gw/GW, n_slices*(gw+1)/GW). */
int tba_debug_stream_launch(tba_context* ctx, int32_t* out);
int tba_debug_prepare_linear_system(tba_context* ctx, double radius);
int tba_debug_schur_matvec(tba_context* ctx, const double* x_cam /*[n_cam*6]*/,
                           const double* x_intr /*[n_group*10]*/,
                           double* y_cam, double* y_intr);
int tba_debug_solve_linear_system(tba_context* ctx, int32_t* cg_iterations,
                                  double* model_cost_change);
int tba_debug_evaluate_step(tba_context* ctx, double* candidate_cost);
int tba_debug_read(tba_context* ctx, int which, double* out, int64_t n);

#ifdef __cplusplus
}
#endif
#endif  /* THEIA_BA_B200_H_ */
