/* b200slam -- C ABI of the Hopper-native scan matcher and SE(2) pose-graph solver.
 *
 * This is the drop-in boundary for the ONE hot path of SteveMacenski/slam_toolbox:
 *   (1) karto::ScanMatcher::MatchScan            (lib/karto_sdk/src/Mapper.cpp:534-639)
 *   (2) the karto::ScanSolver plugin surface     (lib/karto_sdk/include/karto_sdk/Mapper.h:954-1065,
 *       implemented today by solver_plugins::CeresSolver, solvers/ceres_solver.cpp)
 *
 * Plain C: opaque handles, POD structs, HOST pointers in and out, int status codes, no
 * exceptions, no ROS / Eigen / Boost / torch types.  One handle is used by one thread at a
 * time (the reference classes are not re-entrant either: Mapper.h:1496-1503, and every
 * CeresSolver method takes nodes_mutex_).  There is no CPU fallback: every entry point that
 * computes returns B200_ERR_CUDA when no sm_90 device is usable.
 *
 * INTEGRATION.md shows the reference-side bindings (the link-time replacement of
 * ScanMatcher::{Create,MatchScan} and the `class B200Solver : public karto::ScanSolver`
 * plugin adapter) that sit on top of this header.
 */
#ifndef B200SLAM_H
#define B200SLAM_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_INVALID_ARG 1   /* NULL handle / bad sizes / parameters ScanMatcher::Create rejects (Mapper.cpp:481-493) */
#define B200_ERR_CUDA 2          /* no usable device or a CUDA call failed; b200_last_error() has the text */
#define B200_ERR_UNSUPPORTED 3   /* geometry the device path cannot represent (reported, never silently approximated) */
#define B200_ERR_NOT_FOUND 4     /* unknown node / edge id */
#define B200_ERR_NUMERIC 5       /* singular covariance, solver produced no usable solution */

const char * b200_last_error(void);
/* Device selection for handles created afterwards by this thread (cudaSetDevice). */
int b200_set_device(int ordinal);
int b200_device_count(void);
/* The library's host thread pool (B200_HOST_THREADS, default <= 8 threads; it builds lookup tables and descriptor lists), open to
 * the reference-side bindings for host work that sits next to the seam: fn(i, ctx) for i in [0, n), the caller takes part.
 * integration/scan_matcher_b200.cpp uses it for MapperGraph::CorrectPoses' per-scan SetCorrectedPoseAndUpdate (Mapper.cpp:2019-2025). */
void b200_parallel_for(int32_t n, void (*fn)(int32_t, void *), void * ctx);
int32_t b200_host_threads(void);

/* ------------------------------------------------------------------------------------------
 * Scan matcher
 * ---------------------------------------------------------------------------------------- */

/* Everything ScanMatcher::Create (Mapper.cpp:477) takes plus the eight karto::Mapper
 * parameters MatchScan/operator() read at call time (Mapper.cpp:590-594, 626-627, 675-682).
 * The *_variance_penalty fields hold the values as karto STORES them, i.e. already squared
 * by Mapper::setParamDistanceVariancePenalty / AngleVariancePenalty (Mapper.cpp:2562-2570). */
typedef struct b200sm_params {
  double search_size;                 /* CorrelationSearchSpaceDimension / LoopSearchSpaceDimension (m) */
  double resolution;                  /* ...Resolution (m)                                              */
  double smear_deviation;             /* ...SmearDeviation (m)                                          */
  double range_threshold;             /* LaserRangeFinder::GetRangeThreshold() (m) -> grid margin       */
  double coarse_search_angle_offset;  /* rad */
  double coarse_angle_resolution;     /* rad */
  double fine_search_angle_offset;    /* rad; used as the fine angular RESOLUTION (Mapper.cpp:627)      */
  double distance_variance_penalty;
  double angle_variance_penalty;
  double minimum_distance_penalty;
  double minimum_angle_penalty;
  int32_t use_response_expansion;
} b200sm_params;

/* What MatchScan reads from a karto::LocalizedRangeScan (Karto.h:5411-5763). */
typedef struct b200_scan {
  int32_t n;                 /* GetNumberOfRangeReadings()                                             */
  const double * ranges;     /* GetRangeReadings(): n raw readings, NaN/Inf allowed (Karto.h:6869)     */
  const double * points_xy;  /* GetPointReadings(false): n UNFILTERED world points, x,y interleaved    */
  double sensor_pose[3];     /* GetSensorPose(): x, y, heading                                         */
} b200_scan;

/* LocalizedRangeScan::Update (Karto.h:5644-5704): the unfiltered world-frame point readings of a
 * scan, for callers that do not already hold a karto::LocalizedRangeScan. Host libm (glibc) like
 * the reference; out_xy = n x,y pairs. */
int b200_point_readings(const double * ranges, int32_t n, const double sensor_pose[3],
                        double minimum_angle, double angular_resolution, double * out_xy);

typedef struct b200sm b200sm;

/* ScanMatcher::Create. B200_ERR_INVALID_ARG where the reference returns NULL or throws
 * (smear deviation outside [0.5, 10] * resolution, Mapper.h:1226-1235). */
int b200sm_create(const b200sm_params * params, b200sm ** out);
void b200sm_destroy(b200sm * h);
/* Run this handle's kernels on an existing cudaStream_t (e.g. the caller's current stream).
 * NULL (the legacy default stream) = go back to a stream owned by the handle. */
int b200sm_set_stream(b200sm * h, void * cuda_stream);

/* ScanMatcher::MatchScan(pScan, rBaseScans, rMean, rCovariance, doPenalize, doRefineMatch)
 * (Mapper.cpp:534-639).  base[0..nbase) in the order of the reference's scan vector / map
 * (order is part of the contract: SURVEY.md 7, hard part 2).  cov is row-major 3x3.
 * Bounds (this call and b200sm_correlate): a query of at most 51,200 readings (one lookup row of
 * n int32 must fit 200 KB of shared memory; more -> B200_ERR_UNSUPPORTED once the raster is built,
 * before any correlation kernel runs); at most 2^26 poses (nX * nY * nAngles) per pass, split
 * between positions and angles in any way (B200_ERR_INVALID_ARG above that); a correlation ROI narrower than 32,768 cells
 * (b200sm_create returns B200_ERR_UNSUPPORTED otherwise). */
int b200sm_match(b200sm * h, const b200_scan * query, const b200_scan * base, int32_t nbase,
                 int32_t do_penalize, int32_t do_refine, double mean[3], double cov[9],
                 double * response);

/* ScanMatcher::CorrelateScan (Mapper.cpp:712-862) against the grid rasterised by the last
 * b200sm_match / b200sm_raster call. cov is in/out like the reference's rCovariance.
 * If sums != NULL it receives the integer correlation volume, index (y*nX + x)*nAngles + a,
 * and dims = {nX, nY, nAngles}. */
int b200sm_raster(b200sm * h, const b200_scan * query, const b200_scan * base, int32_t nbase);
int b200sm_correlate(b200sm * h, const b200_scan * query, const double center[3],
                     const double search_offset[2], const double search_resolution[2],
                     double angle_offset, double angle_resolution, int32_t do_penalize,
                     int32_t fine, double mean[3], double cov[9], double * response,
                     int32_t * sums, int32_t sums_cap, int32_t dims[3]);

/* ScanMatcher::GetCorrelationGrid() (Mapper.h:1435): geometry + bytes of the last raster.
 * info = width, height, stride, roi_x, roi_y, roi_w, roi_h, data_size, kernel_size. */
int b200sm_grid_info(b200sm * h, int32_t info[9], double offset[2]);
int b200sm_grid_copy(b200sm * h, uint8_t * out, int32_t cap);

/* Batched MatchScan: the loop-closure candidate sweep (Mapper.cpp:1500-1561 calls MatchScan
 * once per candidate chain; here all (query, chain) pairs go to the device together).
 *   scans[0..nscans)            all candidate scans
 *   chain_start[0..nchains]     chain j = scans[chain_start[j] .. chain_start[j+1])
 *   pair_query/pair_chain[np]   pairs to match; both NULL = all nq*nchains pairs, query-major
 * Outputs per pair p: response[p], mean[3p..], cov[9p..]  -- identical to calling
 * b200sm_match(h, &queries[pair_query[p]], chain pair_chain[p], ...) one by one.
 * Bounds (this call and b200sm_batch_upload / _run below): any angle window; a query may have up to
 * 51,200 readings (one lookup row of n int32 must fit 200 KB of shared memory; more -> upload returns
 * B200_ERR_UNSUPPORTED); a candidate scan up to 12,044 readings (FindValidPoints stages 17 B per point in
 * 200 KB of shared memory; more -> run returns B200_ERR_UNSUPPORTED). */
int b200sm_match_batch(b200sm * h, const b200_scan * queries, int32_t nq, const b200_scan * scans,
                       int32_t nscans, const int32_t * chain_start, int32_t nchains,
                       const int32_t * pair_query, const int32_t * pair_chain, int32_t npairs,
                       int32_t do_penalize, int32_t do_refine, double * response, double * mean,
                       double * cov);

/* The same sweep split so that the device part can be timed with inputs resident in HBM:
 *   upload  : host prep (lookup tables) + H2D of queries / candidate scans / pair list
 *   run     : kernels only (asynchronous on the handle's stream); may be repeated
 *   fetch   : D2H of the per-pair results + the libm part of the epilogue
 * kernel_ms: device time of the dominant (correlation) kernel of the last run, from CUDA
 * events recorded on the handle's stream around that launch (blocks until it finished). */
int b200sm_batch_upload(b200sm * h, const b200_scan * queries, int32_t nq, const b200_scan * scans,
                        int32_t nscans, const int32_t * chain_start, int32_t nchains,
                        const int32_t * pair_query, const int32_t * pair_chain, int32_t npairs,
                        int32_t do_penalize);
int b200sm_batch_run(b200sm * h);
int b200sm_batch_fetch(b200sm * h, double * response, double * mean, double * cov);
int b200sm_batch_kernel_ms(b200sm * h, float * ms);
/* per-pair best integer correlation sum and the flat index (y*nX+x)*nA+a of its first
 * arg-max pose from the last run (parity: "integer correlation-grid indices bit-exact") */
int b200sm_batch_best(b200sm * h, int32_t * best_sum, int32_t * best_index, int32_t * tie_count);
/* Multi-GPU sweep (SURVEY.md 8e): writes, for each of the nq queries, the packed key
 *   (best integer correlation sum << 32) | (0xFFFFFFFF - (id_offset + chain index))
 * of this rank's best candidate into device_keys (nq uint64 in DEVICE memory, e.g. the buffer the
 * caller hands to ncclAllReduce(ncclMax) / torch.distributed.all_reduce(MAX) next), on the
 * handle's stream. A max over ranks selects the highest sum, ties to the lowest global id. */
int b200sm_batch_reduce_keys(b200sm * h, void * device_keys, int64_t id_offset);
/* The same exchange without a reduction operator and without host round trips, also valid for penalised sweeps
 * (whose response order is not the integer-sum order): winner_records writes, per query, this rank's best candidate --
 * highest best response, ties to the lowest global id -- with its raw device reduction into device_records
 * (nq records of b200sm_batch_winner_record_bytes() bytes, DEVICE memory, on the handle's stream).  The caller gathers
 * the records of all ranks with ONE collective (ncclAllGather / torch.distributed.all_gather_into_tensor, rank-major),
 * then winners_select picks each query's winner over the nranks x nq gathered records and finishes it (heading
 * average, covariance tail) exactly like batch_fetch does for its own pairs: every rank ends with the same
 * (global id, response, mean[3], cov[9]) per query, bit-identical to the owner's.  winner_id -1 = no candidate. */
int32_t b200sm_batch_winner_record_bytes(void);
int b200sm_batch_winner_records(b200sm * h, void * device_records, int64_t id_offset);
int b200sm_batch_winners_select(b200sm * h, const void * device_gathered, int32_t nranks, int64_t * winner_id,
                                double * response, double * mean, double * cov);
/* Which kernel the uploaded sweep will run on and how its lookups were classified: info = {kernel: 0 generic, 1 single-CTA
 * shared-memory kernel (search <= 48 x 48 poses, grid <= 576 cells), 2 tiled cluster kernel (any search size / range threshold);
 * FAST descriptors, EDGE beams (window leaves the grid), FAR beams (column offset >= one stride), reason code when the
 * shared-memory paths were refused (0 = n/a), CTAs, pairs, items}. */
int b200sm_batch_info(b200sm * h, int32_t info[8]);
/* Plan of the tiled cluster kernel for the uploaded sweep: info = {available, cluster size (CTAs per pair), angle chunks,
 * sub-grid bands per parity phase, rows per band, refusal reason, resident clusters, shared memory per CTA (KB)}. */
int b200sm_batch_tile_info(b200sm * h, int32_t info[8]);
/* Pose-window tiling of the tiled cluster kernel (zero when it was refused): layout = {rows per y-tile (48: six row tiles of 8;
 * 40: five, the window's last row then runs as a tail row), y-tiles, x-tiles, tail row (1 / 0)}. */
int b200sm_batch_tile_layout(b200sm * h, int32_t layout[4]);
/* What the tiled kernel's descriptor blocks hold for the uploaded sweep (host-side counts, zero when the tiled kernel was
 * refused): stats = {descriptor blocks, continuation sub-blocks (a stage's angles split over several staging buffers), largest
 * EDGE group (beams), (angle, phase, band, alignment) groups cut into more than one item, multi entries (cell, multiplicity),
 * largest multiplicity, largest plain group (beams), wrap2 entries}. */
int b200sm_batch_tile_stats(b200sm * h, int32_t stats[8]);
/* The tiled cluster kernel's plan for a geometry, without a handle or a device: in = {grid row stride, grid height, poses in x,
 * poses in y, angles, beams per query, longest candidate scan (readings, rounded up to 4), penalised (1 / 0), pairs, SMs, forced
 * cluster size, minimum angle chunks (0 = automatic), tail layout allowed (1 / 0)}; out = {refusal reason (0 = the kernel runs),
 * cluster size, angle chunks, bands, rows per band, dynamic shared memory per CTA (bytes), tail row (1 / 0)}. */
int b200sm_tile_plan(const int32_t in[13], int32_t out[7]);
/* How the last fetch finished its pairs: stats = {pairs whose volume was all zero (all poses tie: closed form, once per
 * query; with use_response_expansion: pairs with an empty raster, closed form of the widest expansion pass), pairs handed one by one to the single-match path (tie list overflow with a non-zero best, response expansion),
 * pairs, 0}. */
int b200sm_batch_fetch_stats(b200sm * h, int32_t stats[4]);
/* Host wall time (ms) of the last upload: out = {per-query lookup tables (ComputeOffsets), descriptor tables of the kernel, whole call}. */
int b200sm_batch_upload_timing(b200sm * h, double out[3]);
/* bytes copied host->device by upload and device->host by fetch since the last reset */
int b200sm_batch_transfer_bytes(b200sm * h, int64_t * h2d_bytes, int64_t * d2h_bytes, int32_t reset);
/* Tuning / testing switches. "force_generic_sweep" = 1 runs batched sweeps on the generic kernel even
 * where the shared-memory fast path applies; "no_beam_dedup" = 1 keeps one lookup descriptor per beam in the fast
 * path instead of merging beams that hit the same cell; "sweep_kernel" = 0 auto / 1 single-CTA kernel / 2 tiled cluster
 * kernel; "sweep_cluster" = CTAs per pair of the tiled kernel (0 auto, 1, 2, 4, 8); "sweep_chunks" = minimum number of angle chunks (0 auto).
 * All variants produce identical results. */
int b200sm_set_option(b200sm * h, const char * name, int32_t value);
/* Accumulated host wall time (ms) of the single-match path's phases since the last reset: out = {valid points + occupancy
 * replay, raster upload + stamp, lookup-table build, volume (H2D, kernel, D2H, wait), FP64 epilogue, number of matches}. */
int b200sm_match_timing(b200sm * h, double out[6], int32_t reset);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t b200sm_launch_count(const b200sm * h);

/* ------------------------------------------------------------------------------------------
 * SE(2) pose-graph solver  (karto::ScanSolver, Mapper.h:954-1065)
 * ---------------------------------------------------------------------------------------- */

/* The knobs CeresSolver::Configure sets (solvers/ceres_solver.cpp:96-186); defaults from
 * b200pg_default_opts() reproduce them. */
typedef struct b200pg_opts {
  int32_t max_num_iterations;        /* Ceres default 50                                        */
  double function_tolerance;         /* 1e-3  (ceres_solver.cpp:158)                            */
  double gradient_tolerance;         /* 1e-6  (:159)                                            */
  double parameter_tolerance;        /* 1e-3  (:160)                                            */
  double min_relative_decrease;      /* 1e-3  (:171)                                            */
  double initial_trust_region_radius;/* 1e4   (:173)                                            */
  double max_trust_region_radius;    /* 1e8   (:174)                                            */
  double min_trust_region_radius;    /* 1e-16 (:175)                                            */
  double min_lm_diagonal;            /* 1e-6  (:177)                                            */
  double max_lm_diagonal;            /* 1e32  (:178)                                            */
  int32_t jacobi_scaling;            /* 1     (:169)                                            */
  int32_t use_nonmonotonic_steps;    /* 1     (:164)                                            */
  int32_t max_consecutive_nonmonotonic_steps; /* 3 (:165)                                       */
  int32_t max_num_consecutive_invalid_steps;  /* 3 (:163)                                       */
  /* linear solver (replaces SPARSE_NORMAL_CHOLESKY, :100-102): block-Jacobi PCG on the
   * normal equations, iterated to ||r|| <= pcg_tolerance * ||b|| */
  double pcg_tolerance;              /* 1e-9: poses stay within 5e-6 m / 5e-7 rad of the exact-solve LM on cfg4 (1e-8 would not);
                                      * under dogleg the Gauss-Newton solve runs to pcg_tolerance / 10 */
  int32_t pcg_max_iterations;        /* 20000 */
  /* ceres_loss_function (ceres_solver.cpp:82-94): 0 = none (squared loss, the default), 1 = HuberLoss(loss_scale),
   * 2 = CauchyLoss(loss_scale); the reference uses scale 0.7 for both */
  int32_t loss_function;
  double loss_scale;                 /* 0.7 */
  /* ceres_trust_strategy (ceres_solver.cpp:46-58): 0 = LEVENBERG_MARQUARDT (the default), 1 = DOGLEG.
   * ceres_dogleg_type (:138-155), read with DOGLEG only: 0 = TRADITIONAL_DOGLEG, 1 = SUBSPACE_DOGLEG.
   * Other values are refused with B200_ERR_INVALID_ARG. */
  int32_t trust_region_strategy;
  int32_t dogleg_type;
  /* linear solver of every trust-region step: 0 = the PCG kernels above (the default), 1 = exact block-sparse Cholesky
   * (SPARSE_NORMAL_CHOLESKY, ceres_solver.cpp:96-97): an FP64 supernodal factorisation of (H + shift D^2) over the free
   * nodes on the device, after a host analysis that is kept while the free nodes and their adjacent pairs stay the same.
   * pcg_tolerance and pcg_max_iterations do not apply to it. Other values are refused with B200_ERR_INVALID_ARG. */
  int32_t linear_solver_type;
} b200pg_opts;
/* b200pg_opts and b200pg_summary grew (trust_region_strategy, dogleg_type, linear_solver_type; linear_solves): the ctypes
 * mirror (slam_toolbox_b200/api.py PgOpts / PgSummary) and every compiled caller must be rebuilt against this header. */

typedef struct b200pg_summary {
  int32_t iterations;          /* LM iterations (successful + unsuccessful)            */
  int32_t successful_steps;
  int32_t pcg_iterations;      /* total over all LM iterations                         */
  int32_t termination;         /* 0 convergence(function) 1 gradient 2 parameter 3 max-iter 4 min-radius 5 failure */
  int32_t usable;              /* ceres::Solver::Summary::IsSolutionUsable()           */
  double initial_cost, final_cost;
  float solve_ms;              /* device time of the whole solve (CUDA events)         */
  int64_t kernel_launches;
  float setup_ms;              /* host time before the first kernel: flatten / adjacency / uploads of what changed */
  float wall_ms;               /* host wall time of the whole call                     */
  int32_t uploaded_edges;      /* constraints copied to the device by this call (the ones added since the last solve) */
  int32_t linear_solver;       /* PCG kernel the plan chose: 0 global block-Jacobi, 1 shared-memory block-Jacobi,
                                * 3 two-level with 3 coarse modes, 6 two-level with 6 coarse modes, 13 / 16 the same
                                * two-level preconditioner with 3 / 6 coarse modes on global-memory aggregates and a dense
                                * coarse inverse (graphs too large for 3 / 6); 8 block-sparse Cholesky
                                * (linear_solver_type = 1, pcg_iterations stays 0); -1 no linear solve planned */
  int32_t linear_solves;       /* PCG solves or Cholesky factorisations this call ran, retries at a larger regulariser
                                * included: one per iteration under LM; under dogleg none for an iteration that reuses the
                                * Gauss-Newton step. setup_ms includes the Cholesky analysis when one ran */
} b200pg_summary;

typedef struct b200pg b200pg;

void b200pg_default_opts(b200pg_opts * o);
int b200pg_create(const b200pg_opts * opts_or_null, b200pg ** out);
void b200pg_destroy(b200pg * h);
int b200pg_set_stream(b200pg * h, void * cuda_stream);
/* CeresSolver::Configure (solvers/ceres_solver.cpp:25-193) runs after construction: replace / read the options of a live handle
 * (the graph is kept). */
int b200pg_set_opts(b200pg * h, const b200pg_opts * opts);
int b200pg_get_opts(const b200pg * h, b200pg_opts * opts);
/* ScanSolver::Reset (Mapper.h:1028; ceres_solver.cpp:272-314): drop everything, un-fix the anchor */
int b200pg_reset(b200pg * h);
/* ScanSolver::Clear (Mapper.h:1021): drop the corrections of the last solve only */
int b200pg_clear(b200pg * h);
/* ScanSolver::AddNode (ceres_solver.cpp:317-336): id = scan UniqueId, pose = corrected pose.
 * The first node ever added becomes the gauge anchor (:333-335). */
int b200pg_add_node(b200pg * h, int32_t id, const double pose[3]);
/* ScanSolver::AddConstraint (ceres_solver.cpp:339-392): z = LinkInfo::GetPoseDifference(),
 * cov = LinkInfo::GetCovariance() (row-major). The library forms the sqrt-information
 * U = chol(cov^-1).matrixU() like :364-376. Unknown or identical nodes are refused silently
 * in the reference (returns B200_ERR_NOT_FOUND here, state unchanged). */
int b200pg_add_edge(b200pg * h, int32_t id_a, int32_t id_b, const double z[3], const double cov[9]);
int b200pg_remove_node(b200pg * h, int32_t id);                 /* ceres_solver.cpp:395-425 */
int b200pg_remove_edge(b200pg * h, int32_t id_a, int32_t id_b); /* :428-448, either orientation */
/* ScanSolver::ModifyNode (:451-461): sets x,y and ADDS the stored yaw to pose[2]. */
int b200pg_modify_node(b200pg * h, int32_t id, const double pose[3]);
int b200pg_get_node(const b200pg * h, int32_t id, double pose[3]);  /* getGraph / GetNodeOrientation */
int32_t b200pg_num_nodes(const b200pg * h);
int32_t b200pg_num_edges(const b200pg * h);
/* ScanSolver::Compute (:214-269): solves in place. On an unusable solution the node store
 * and corrections are left untouched and B200_ERR_NUMERIC is returned. */
int b200pg_solve(b200pg * h, b200pg_summary * summary_or_null);
/* ScanSolver::GetCorrections (Mapper.h:988): all nodes after the last solve; returns count
 * written (<= cap). Empty after b200pg_clear(). */
int32_t b200pg_get_corrections(const b200pg * h, int32_t * ids, double * poses, int32_t cap);
/* The host analysis of the Cholesky linear solver, stateless and without a device: nodes 0..n-1, edges [e][2] node
 * indices, fixed = the constant node or -1. The free nodes are the ones in some edge, except fixed. info = {free block
 * columns, nonzero 3x3 blocks of L (diagonal included), supernodes, supernodal critical-path length, widest supernode
 * (block columns), tallest panel (block rows), factor flops (sum over scalar columns of the squared column count), 0};
 * order (may be NULL, else cap >= free nodes) receives the free nodes in elimination order. The ordering is a function of
 * the free nodes and the set of adjacent pairs alone. A solve with linear_solver_type = 1 runs this same analysis. */
int b200pg_cholesky_analyze(int32_t n, int32_t e, const int32_t * edge_nodes, int32_t fixed, int64_t info[8], int32_t * order,
                            int32_t cap);
/* The info record of the analysis the handle's last Cholesky solve used (zeros when there was none), with info[7] = the
 * analyses this handle has run. */
int b200pg_factor_info(const b200pg * h, int64_t info[8]);

/* ------------------------------------------------------------------------------------------
 * Occupancy grid: karto::OccupancyGrid::CreateFromScans (Karto.h:5946-5961), the map-publish step
 * next to the hot path (slam_toolbox: SMapper::getOccupancyGrid src/slam_mapper.cpp:63-69, called
 * from SlamToolbox::updateMap src/slam_toolbox_common.cpp:630-654 with ALL processed scans).
 *
 * The scans live in HBM behind the handle: append them as the mapper processes them (or re-load
 * them after a loop closure moved their poses), then build as often as a map is wanted.  A build
 * is: bounding box of the scans (ComputeDimensions Karto.h:6082-6107) -> one Bresenham trace per
 * beam into the pass / hit counters (AddScan Karto.h:6139-6182, RayTrace :6193-6229, TraceLine
 * :4874-4927) -> cell states (Update :6259-6274).  Counters are integers, so the result is
 * bit-identical to the reference's whatever the order the beams are traced in.
 * ---------------------------------------------------------------------------------------- */
#define B200_CELL_UNKNOWN 0      /* GridStates_Unknown  Karto.h:4379 */
#define B200_CELL_OCCUPIED 100   /* GridStates_Occupied Karto.h:4380 */
#define B200_CELL_FREE 255       /* GridStates_Free     Karto.h:4381 */

/* The three laser fields are the DEFAULT limits: those of every scan added by b200og_add_scans (or with a NULL laser
 * array).  A scan added by b200og_add_scans_lasers carries its own limits, as the reference reads each scan's own
 * pScan->GetLaserRangeFinder() (Karto.h:6146-6151, :5646-5698). */
typedef struct b200og_params {
  double resolution;           /* m per cell (CreateFromScans' argument); 0 is rejected (Karto.h:5916-5918) */
  double range_threshold;      /* LaserRangeFinder::GetRangeThreshold(): longer readings are traced up to it, without a hit */
  double minimum_range;        /* LaserRangeFinder::GetMinimumRange(): readings <= it are ignored (Karto.h:6160) */
  double maximum_range;        /* LaserRangeFinder::GetMaximumRange(): readings >= it are ignored              */
  uint32_t min_pass_through;   /* OccupancyGrid "MinPassThrough", 2   (Karto.h:5921, :6241) */
  double occupancy_threshold;  /* OccupancyGrid "OccupancyThreshold", 0.1 (Karto.h:5922, :6246) */
} b200og_params;

typedef struct b200og_info {
  int32_t width, height;       /* Round(bounding-box size / resolution) (Karto.h:6103-6105) */
  int32_t stride;              /* width step: width aligned up to 8 (Karto.h:4640); rows of every array below */
  double offset[2];            /* world position of cell (0,0) = bounding-box minimum (Karto.h:6106) */
} b200og_info;

typedef struct b200og b200og;

/* Karto's defaults for everything but the laser limits (12 m / 0.1 m / 30 m here, SURVEY.md 8d) */
void b200og_default_params(b200og_params * p);
int b200og_create(const b200og_params * params, b200og ** out);
void b200og_destroy(b200og * h);
int b200og_set_stream(b200og * h, void * cuda_stream);
/* The scan store.  add = copy n scans (ranges, unfiltered point readings, sensor position) to the
 * device, after the scans already there; clear = forget them all. */
int b200og_add_scans(b200og * h, const b200_scan * scans, int32_t n);
/* One scan's laser limits, the values of its karto::LaserRangeFinder (see b200og_params). */
typedef struct b200og_laser {
  double range_threshold, minimum_range, maximum_range;
} b200og_laser;
/* b200og_add_scans with per-scan limits: lasers[i] belongs to scans[i] and is stored with it (24 B per scan on the
 * device); builds, range builds, stored boxes and removals use each scan's own limits, so one store may hold the scans of
 * several lasers.  lasers == NULL = the handle's params for every scan (b200og_add_scans is this call with NULL).
 * B200_ERR_INVALID_ARG, with the store unchanged, for a non-finite limit. */
int b200og_add_scans_lasers(b200og * h, const b200_scan * scans, int32_t n, const b200og_laser * lasers);
int b200og_clear_scans(b200og * h);
int32_t b200og_num_scans(const b200og * h);
/* CreateFromScans over the stored scans.  With no scans the reference returns NULL: here
 * B200_ERR_NOT_FOUND, *info zeroed.  B200_ERR_UNSUPPORTED when width step * height exceeds 2^31-1
 * (the reference's kt_int32s data size overflows there too). */
int b200og_build(b200og * h, b200og_info * info);
/* Result of the last build, each array stride * height, any pointer may be NULL:
 * cells = the grid's bytes (B200_CELL_*), pass / hits = the counters behind them. */
int b200og_fetch(b200og * h, uint8_t * cells, uint32_t * pass, uint32_t * hits);
/* the same bytes as a nav_msgs/OccupancyGrid payload (width * height, row-major, -1 / 100 / 0:
 * vis_utils::toNavMap include/slam_toolbox/visualization_utils.hpp:108-146) */
int b200og_fetch_nav(b200og * h, int8_t * data);
/* device time of the last build's kernels (ms) and the kernels it launched */
int b200og_kernel_ms(b200og * h, float * ms);
int64_t b200og_launch_count(const b200og * h);
/* The static entry point in one call: create + add_scans + build.  *out stays NULL (and the call
 * returns B200_ERR_NOT_FOUND) for n == 0, like the reference's NULL. */
int b200og_create_from_scans(const b200og_params * params, const b200_scan * scans, int32_t n, b200og_info * info,
                             b200og ** out);

/* Map merge (slam_toolbox's merge_maps_kinematic, src/merge_maps_kinematic.cpp): the submaps' scans stay in the store and are
 * corrected in place.
 *
 * transform_scans = MergeMapsKinematic::transformScan (:195-248) on scans [first, first + count), one correction given as
 * tf2 holds it (basis row-major 3x3, origin x, y, z).  Every unfiltered point p and the sensor position become
 * ((b[r][0]*x + b[r][1]*y) + b[r][2]*0) + o[r] for r = 0, 1 (tf2::Transform applied to (x, y, 0), unfused), and each
 * scan's stored bounding box becomes the box of its four corrected corners (min, max, (max x, min y), (min x, max y)).
 * Corrections compound: a second call transforms the already transformed scans, as the tool's repeated merges do.
 * sensor_poses = count x 3 host-computed sensor poses for lasers with a mounting offset (only x, y are kept); NULL = the
 * formula above (exact for a laser at the robot origin).  B200_ERR_INVALID_ARG for a range outside the store or a
 * non-finite basis / origin.  After the first transform, every build sizes its grid from the union of the stored boxes
 * (ComputeDimensions reads them: the tool clears IsDirty); before it, a build computes the box from the points as always. */
int b200og_transform_scans(b200og * h, int32_t first, int32_t count, const double basis[9], const double origin[3],
                           const double * sensor_poses);
/* b200og_build over scans [first, first + count) only (one submap's own grid from the shared store); the same results
 * contract.  B200_ERR_NOT_FOUND for count == 0, B200_ERR_INVALID_ARG for a range outside the store. */
int b200og_build_range(b200og * h, int32_t first, int32_t count, b200og_info * info);
/* Per-scan bounding boxes of scans [first, first + count), boxes = count x {min x, min y, max x, max y}: LocalizedRangeScan::
 * Update's box (sensor position + points whose range is within [minimum_range, range_threshold]) until a transform
 * replaced it.  b200og_clear_scans drops the boxes and the transformed state. */
int b200og_scan_boxes(b200og * h, int32_t first, int32_t count, double * boxes);

/* Removes the scans at store indices indices[0 .. n) (strictly increasing) and compacts the store on the device: the
 * survivors keep their order, and every later call sees exactly the store a fresh handle loaded with the surviving scans
 * (their transformed values, after a transform) would hold, so builds give bit-identical grids.  Stored boxes and the
 * transformed state are kept.  Only scans after the first removed one move.  n == 0 does nothing; removing every scan
 * leaves an empty store.  B200_ERR_INVALID_ARG, with the store unchanged, for a NULL indices with n > 0, n < 0, an index
 * outside the store, or indices not strictly increasing.  b200og_kernel_ms reads the compaction kernel's time afterwards.
 * The first removal that moves scans allocates a second copy of the store's device arrays (the compaction target, swapped
 * with the store after each removal) and keeps it for the handle's life: the store's device footprint doubles. */
int b200og_remove_scans(b200og * h, const int32_t * indices, int32_t n);

#ifdef __cplusplus
}
#endif
#endif /* B200SLAM_H */
