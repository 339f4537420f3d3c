/*
 * fcma_b200.h — C ABI of the Hopper-native FCMA correlation engine (libfcma_b200.so).
 *
 * Drop-in boundary for the native modules of brainiak/brainiak @ 123f6e1 on the FCMA hot path:
 *
 *   reference native entry point (file:line)                           replaced by
 *   ------------------------------------------------------------------ ----------------------------
 *   cython_blas.compute_self_corr_for_voxel_sel  cython_blas.pyx:20    fcma_corr_block (layout 0)
 *   cython_blas.compute_corr_vectors             cython_blas.pyx:388   fcma_corr_block (layout 1)
 *   cython_blas.compute_kernel_matrix            cython_blas.pyx:118   fcma_kernel_matrices
 *   cython_blas.compute_single_matrix_multiplication  pyx:480          fcma_gemm_nt
 *   fcma_extension.normalization                 fcma_extension.cc:29  fcma_within_subject_norm
 *   preprocessing._separate_epochs (z-score)     preprocessing.py:80   fcma_pack_operand(normalize=1)
 *   VoxelSelector._voxel_scoring stages 1-3      voxelselector.py:467  fcma_voxel_kernels
 *   VoxelSelector._worker task loop, one mask    voxelselector.py:255  fcma_voxel_kernels_sym  (raw_data2 is None,
 *                                                (+ :289-291)          uses corr[i][e][j] == corr[j][e][i])
 *   Classifier._compute_kernel_matrix_in_portion classifier.py:279     fcma_classifier_kernel
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only.  Pointers named *_dev are CUDA device pointers
 *     (e.g. torch.Tensor.data_ptr()); `stream` is a cudaStream_t passed as void* (0 = default).
 *   - The caller owns every buffer (as in the reference, voxelselector.py:307, classifier.py:166);
 *     the library never retains pointers across calls.
 *   - An entry point writes only the outputs it documents, within their documented extents, and never writes its
 *     const inputs or host arrays; every copy, memset, scratch allocation and launch it issues (uploads of host arrays
 *     such as fold structs, centres, gammas and training masks included) goes on `stream`.
 *   - Return value: 0 on success, negative FCMA_E* on failure; fcma_last_error() returns a
 *     thread-local message.  (Reference: ValueError from Cython memoryviews, RuntimeError from
 *     fcma_extension.cc:47 — the Python wrapper maps FCMA_EINVAL->ValueError, others->RuntimeError.)
 *   - There is NO CPU fallback: every compute entry point fails with FCMA_ENODEV without a
 *     Hopper (sm_90) device.
 */
#ifndef FCMA_B200_H
#define FCMA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FCMA_OK        0
#define FCMA_EINVAL   -1   /* bad argument (-> ValueError)               */
#define FCMA_ECUDA    -2   /* CUDA runtime / driver error (-> RuntimeError) */
#define FCMA_ENODEV   -3   /* no sm_90 device                             */
#define FCMA_ENOMEM   -4   /* scratch buffer too small                    */

/* Operand precision of the correlation contraction (accumulation is always fp32). */
#define FCMA_PREC_BF16     0  /* 1 bf16 plane            : |dr| ~ 1e-3                      */
#define FCMA_PREC_TF32     1  /* 1 tf32 plane            : |dr| ~ 1e-4                      */
#define FCMA_PREC_BF16X3   2  /* bf16 hi/lo, 3 products  : |dr| ~ 1e-6                      */
#define FCMA_PREC_TF32X3   3  /* tf32 hi/lo, 3 products  : fp32-equivalent (|dr| ~ 1e-7)    */
#define FCMA_PREC_F32SIMT  4  /* FFMA reference kernel on the raw fp32 epochs (no packing)  */
#define FCMA_PREC_FP16X3   5  /* fp16 hi/lo (pre-scaled by 2^6), 3 products: fp32-equivalent for
                                 normalised data (|x| <= 1) at bf16 tensor speed               */

/* flags for the fused pipelines */
#define FCMA_FLAG_MASK_SELF      1  /* zero the self-correlation column after normalisation   */
#define FCMA_FLAG_FISHER_IN_PASS2 2 /* Fisher-z in the normalise kernel (default: GEMM epilogue) */
#define FCMA_FLAG_F16_INTERMEDIATE 4 /* round the internal Fisher-z block of the fused pipelines to fp16 (half the
                                        HBM traffic of both kernels; max|dK|/max|K| ~ 1.5e-5 at V2 = 50 000;
                                        always on for the single-product operand modes bf16 / tf32)            */

/* alternate code paths with the SAME results (up to the order of fp32 partial sums), selectable per call so that tests
 * can compare them; the library never reads the environment */
#define FCMA_FLAG_STRIDED_BLOCK   8   /* fused pipelines: strided [nb][E][ld] correlation block instead of the tiled one */
#define FCMA_FLAG_SYM_TRANSPOSED 16   /* symmetric pipeline: store a transposed copy of every block + row pass over it
                                         instead of the column-direction pass (the default for E > 32)               */
#define FCMA_FLAG_COLS_TMA       32   /* column-direction pass fed by 5-D TMA bricks + an mbarrier ring instead of cp.async +
                                         block barriers (needs E % 4 == 0; not the default)                            */
#define FCMA_FLAG_COLS_V2        64   /* column-direction pass of the fp32 block, version 2: thread-per-row normalisation
                                         (no shuffles), fp16 staging, ldmatrix fragments -- half the instructions; not
                                         the default                                                                    */
#define FCMA_FLAG_COLS_PAD32    128   /* E <= 16: column-direction pass with the 32-epoch (padded) kernel instead of the
                                         16-epoch one                                                                   */
#define FCMA_FLAG_COLS_WIDE     256   /* 32 < E <= 64, fp32 block: column-direction pass (k_norm_syrk_cols64: one column voxel
                                         per warp, 8-column strips) instead of the transposed copy: half the scratch per block
                                         row; not the default                                                           */

int         fcma_version(void);
const char *fcma_last_error(void);
/* number of usable sm_90 devices (0 if none); never fails */
int         fcma_device_count(void);

/* ---- operand packing (+ optional a14 normalise prologue) ---------------------------------- */
/* K extent (elements per voxel row per plane) of a packed operand for epochs of length T. */
int    fcma_operand_kp(int precision, int T);
/* planes of a packed operand (1 or 2) */
int    fcma_operand_planes(int precision);
/* bytes of a packed operand: [planes][E][V][Kp] (rounded up to 256 B) followed by the exact
 * self-correlation diagonal [E][V] float32 (sequential-FMA sum of squares, see DESIGN.md §5) */
size_t fcma_operand_bytes(int precision, int E, int T, long V);

/* epochs_dev: float32 [E][T][ld] (voxels contiguous, row pitch ld >= V; rows t >= T_e[e] must be
 * zero when T_e differs per epoch).  T_e: host array of E epoch lengths or NULL (= all T).
 * normalize: 0 = data already normalised (reference contract, voxelselector.py:72-76);
 *            1 = apply preprocessing.py:80-84 per epoch (z-score over the T_e rows, nan->0, /sqrt(T_e)).
 * Writes the K-major, precision-split operand [planes][E][V][Kp] (+ diagonal) into packed_dev. */
int fcma_pack_operand(const float *epochs_dev, int E, int T, long V, long ld, const int *T_e,
                      int normalize, int precision, void *packed_dev, size_t packed_bytes,
                      void *stream);

/* same for the voxels [v_begin, v_end) only, written to their places in the V-voxel operand: a shard of the symmetric
 * pipeline that starts at row s only ever touches voxels >= s (rows [s, s+n) against columns [s, V)) */
int fcma_pack_operand_range(const float *epochs_dev, int E, int T, long V, long ld, const int *T_e,
                            int normalize, int precision, long v_begin, long v_end, void *packed_dev,
                            size_t packed_bytes, void *stream);

/* a14 alone, in place on float32 [E][T][ld] (preprocessing.py:80-84). */
int fcma_epoch_normalize(float *epochs_dev, int E, int T, long V, long ld, const int *T_e,
                         void *stream);

/* ---- a4 / a9: correlation block -------------------------------------------------------------- */
/* out[i*stride_i + e*stride_e + j] = sum_t rows[e][t][start+i] * cols[e][t][j]
 *   i < nb, e < E, j < V2.   layout 0 ([nb,E,V2]): stride_i = E*ld, stride_e = ld;
 *                            layout 1 ([E,nb,V2]): stride_i = ld,   stride_e = nb*ld   (ld >= V2).
 * rows_op / cols_op: packed operands (same precision) of raw_data [.,.,V] and raw_data2 [.,.,V2]
 * (pass the same pointer for self-correlation).  fisher_epochs: epochs e < fisher_epochs get
 * 0.5*log((1+r)/(1-r)) with the clamps of fcma_extension.cc:68-72 applied in the epilogue; 0 = raw r. */
int fcma_corr_block(const void *rows_op, const void *cols_op, int precision, int E, int T, long V,
                    long V2, long start, long nb, float *out_dev, long stride_i, long stride_e,
                    int fisher_epochs, void *stream);

/* same contraction with fp32 FFMA on the unpacked epochs [E][T][ld*] (reference-order numerics) */
int fcma_corr_block_f32(const float *rows_epochs, long ldr, const float *cols_epochs, long ldc,
                        int E, int T, long V, long V2, long start, long nb, float *out_dev,
                        long stride_i, long stride_e, void *stream);

/* ---- a6: Fisher-z + within-subject z-score, in place (exact semantics of fcma_extension.cc:52-84,
 * including untouched trailing epochs); corr: float32 [n0][E][n2] contiguous. */
int fcma_within_subject_norm(float *corr_dev, long n0, int E, long n2, int eps, void *stream);

/* ---- a7 / a11: linear kernels ------------------------------------------------------------------ */
/* K[i] = beta*K[i] + Z_i Z_i^T, Z_i = z[i*stride_i + e*ld + j], j < n2; K: [nb][E][E] (full, symmetric).
 * With sum_over_rows != 0 a single [E][E] matrix K = beta*K + sum_i Z_i Z_i^T is produced
 * (Classifier, classifier.py:334-339). */
int fcma_kernel_matrices(const float *z_dev, long nb, int E, long n2, long stride_i, long ld,
                         float beta, float *K_dev, int sum_over_rows, void *stream);

/* fused a6+a7: input is raw r (fisher_done=0) or Fisher-z for epochs < (E/eps)*eps (fisher_done=1);
 * normalised values are never written.  self_col0 >= 0: column of voxel 0's self-correlation
 * (voxel i masks column self_col0+i), -1: no masking. */
int fcma_norm_kernel_matrices(const float *corr_dev, long nb, int E, long n2, long stride_i, long ld,
                              int eps, int fisher_done, long self_col0, float beta, float *K_dev,
                              int sum_over_rows, void *stream);

/* ---- fused pipelines ----------------------------------------------------------------------------- */
/* bytes of scratch needed per block row by the pipelines (so callers can size `work`) */
size_t fcma_work_bytes_per_row(int E, long V2);

/* a4 -> a6 -> a7 for voxel rows [start, start+nb): K_dev[nb][E][E] (unshrunk; the decimal shrink of
 * voxelselector.py:409-412 is applied by the caller).  work_dev: scratch of work_bytes
 * (>= fcma_work_bytes_per_row; more rows per pass = fewer launches). */
int fcma_voxel_kernels(const void *rows_op, const void *cols_op, int precision, int E, int T, long V,
                       long V2, long start, long nb, int eps, int flags, float *work_dev,
                       size_t work_bytes, float *K_dev, void *stream);

/* Replaces the worker's whole task loop (voxelselector.py:255-282 over _voxel_scoring, :467-516) when raw_data2 is None
 * (:289-291).  Same result for SELF-correlation at half the tensor work, using corr[i][e][j] == corr[j][e][i]:
 * rows [start, start+nb) are contracted with columns [start, V) only and every block is used twice, for its row
 * voxels and (transposed) for its column voxels.  K_dev is the FULL [V][E][E] array and is ACCUMULATED into
 * (caller zeroes it): after this call K[i] (start <= i < start+nb) holds the columns j >= start, and K[j]
 * (j >= start+nb) has received the columns in [start, start+nb); rows i < start are not touched.  Calling it once
 * with (0, V), or once per shard of a partition of [0, V) -- e.g. one shard per GPU followed by a sum (all-reduce) of
 * the K arrays -- yields the same kernels as fcma_voxel_kernels.  nb must be a multiple of 256 unless start+nb == V;
 * eps a power of two (fused path); work_dev must hold at least 256 rows (see fcma_sym_rows_per_pass). */
int fcma_voxel_kernels_sym(const void *op, int precision, int E, int T, long V, long start, long nb, int eps,
                           int flags, float *work_dev, size_t work_bytes, float *K_dev, void *stream);
/* The same for epochs that are still arriving (multi-GPU input exchange): epochs_dev receives `ngroups` contiguous epoch
 * groups [e0[g], e0[g] + cnt[g]); ready_events[g] is a cudaEvent_t (NULL: already there) that fires when group g is complete.
 * The library packs each group into op_dev (voxels [start, V) only) once its event has fired and runs the GEMMs of the first
 * pass -- of the first two passes if work_dev holds two blocks -- group by group, hiding the upload; then as above. */
int fcma_voxel_kernels_sym_grouped(const float *epochs_dev, const int *T_e, int normalize, void *op_dev, size_t op_bytes,
                                   int precision, int E, int T, long V, long start, long nb, int eps, int flags,
                                   int ngroups, const int *e0, const int *cnt, void *const *ready_events,
                                   float *work_dev, size_t work_bytes, float *K_dev, void *stream);
/* 1 if fcma_voxel_kernels_sym takes the column voxels' sums from the stored block itself (column-direction
 * normalise+SYRK pass: E <= 32, power-of-two eps <= 32; fp32 or fp16 block), 0 if it stores a transposed copy of
 * every block and runs the row pass over it (E > 32).  Informational (bench accounting, scratch sizing). */
int fcma_sym_uses_column_pass(int precision, int E, int eps, int flags);
/* voxel rows fcma_voxel_kernels_sym takes per pass with a scratch buffer of work_bytes (a multiple of 256; < 256 means
 * the buffer is too small): the column-pass variant keeps only the block itself, the other one also its transposed copy */
long fcma_sym_rows_per_pass(int precision, int E, int eps, int flags, long V, long start, size_t work_bytes);

/* a9 -> a10 -> a11: K_dev[E][E] += sum over rows [start, start+nb) (beta = 1 semantics, caller zeroes
 * K first as classifier.py:311-313 does); eps <= 1 skips the normalisation (classifier.py:204). */
int fcma_classifier_kernel(const void *rows_op, const void *cols_op, int precision, int E, int T,
                           long V, long V2, long start, long nb, int eps, int flags, float *work_dev,
                           size_t work_bytes, float *K_dev, void *stream);

/* The same for ONE mask (rows == columns == all V voxels, eps >= 2 a power of two, E <= 64) on the symmetric GEMM: every
 * voxel pair is contracted once, K_dev[E][E] += sum over all pairs -- row passes only (diagonal squares once, the blocks
 * right of them twice), fp64 accumulation on the device.  work_dev: at least 256 rows of fcma_work_bytes_per_row(E, V). */
int fcma_classifier_kernel_sym(const void *op, int precision, int E, int T, long V, int eps, int flags,
                               float *work_dev, size_t work_bytes, float *K_dev, void *stream);

/* ---- a7 tail + a8 on the GPU (SURVEY §8f rank 1) ------------------------------------------------ */
/* decimal shrink of voxelselector.py:409-412 on every [E][E] kernel, in place; digits_dev (optional,
 * int[nv]) receives len(str(int(K[0][0]))) */
int fcma_shrink_kernels(float *K_dev, long nv, int E, int *digits_dev, void *stream);

/* the kernels of a subset of the epochs, out of place: out_dev[v][a][b] = K_dev[v][keep[a]][keep[b]], a contiguous
 * [nv][E_keep][E_keep] array (leave-one-subject-out: the full run's kernels without one subject's rows and columns).
 * keep_host: E_keep strictly increasing epoch indices in [0, E), E <= 256, read on the host and passed to the kernel by
 * value.  shrink != 0 also applies fcma_shrink_kernels' decimal shrink, its digits counted on the compacted
 * out[v][0][0]; digits_dev (optional, int[nv]) receives them.  The output must not overlap K_dev. */
int fcma_subset_kernels(const float *K_dev, long nv, int E, const int *keep_host, int E_keep, float *out_dev,
                        int shrink, int *digits_dev, void *stream);
/* the same gather on fp64 kernels (K_fit, K_pred, G and D of the feature route), without a shrink */
int fcma_subset_kernels_f64(const double *K_dev, long nv, int E, const int *keep_host, int E_keep, double *out_dev,
                            void *stream);

/* batched cross-validation of SVC(kernel='precomputed') (binary C-SVC, libsvm SMO restated from
 * scikit-learn's sklearn/svm/src/libsvm/svm.cpp) on nv kernels [E][E]: folds_host points to nfolds
 * structs {int n_train, n_pos, n_test, pad; int train_idx[64]; int test_idx[64]; unsigned char test_pos[64]}
 * (training samples of the smaller label first = class +1, as svm_group_classes orders them);
 * correct_dev[v*nfolds + f] = number of correctly predicted held-out samples; iters_dev optional.
 * E <= 64, at most 4096 fold problems, 2 <= n_train <= 64, n_test <= 64.  Replaces voxelselector.py:41-53 (_cross_validation_for_one_voxel)
 * as called by _do_cross_validation (voxelselector.py:423-465) for SVC(kernel='precomputed', shrinking=False).
 * max_iter, here and in the two entry points below, is scikit-learn's SVC(max_iter): at most max_iter SMO iterations per
 * problem, 0 runs none (every alpha stays 0, so rho = 0 and every decision is 0: the second class), and a negative value
 * (-1) means no limit.  The held-out decisions sum alpha_k y_k K(t, k) sequentially in training order and rho sums the
 * free variables in libsvm's order, so the decision values equal libsvm's bit for bit. */
int fcma_svm_cv_precomputed(const float *K_dev, long nv, int E, int nfolds, const void *folds_host, double C,
                            double tol, int max_iter, int *correct_dev, int *iters_dev, void *stream);

/* the general form of the solver.  shrinking != 0: libsvm's shrinking heuristic restated as well (do_shrinking, be_shrunk,
 * reconstruct_gradient, the counter / unshrink logic of Solver::Solve) = scikit-learn's default SVC(shrinking=True).
 * correct_dev and bits_dev are both optional (at least one), iters_dev as well; a null output is not written and the
 * others do not depend on which are given: bit t of bits_dev[v*nproblems + p] is set when sample test_idx[t]
 * of problem p falls on the side of the first (smaller-label) class.  One struct per (fold, class pair) gives one-vs-one
 * multi-class cross-validation (votes as in libsvm's svm_predict: first maximum wins). */
int fcma_svm_cv_solve(const float *K_dev, long nv, int E, int nproblems, const void *folds_host, double C, double tol,
                      int max_iter, int shrinking, int *correct_dev, unsigned long long *bits_dev, int *iters_dev,
                      void *stream);
/* the same solver on fp64 kernels [nv][E][E]: Q_ab = (float)(y_a y_b K_fit_ab), QD_a = K_fit_aa and the decisions
 * sum_k alpha_k y_k K_pred[t][k] - rho in double -- what libsvm computes for a non-precomputed kernel.  K_pred_dev may
 * equal K_fit_dev (linear kernel). */
int fcma_svm_cv_solve_f64(const double *K_fit_dev, const double *K_pred_dev, long nv, int E, int nproblems,
                          const void *folds_host, double C, double tol, int max_iter, int shrinking, int *correct_dev,
                          unsigned long long *bits_dev, int *iters_dev, void *stream);
/* fcma_svm_cv_solve for wider problems, on float kernels [nv][E][E] with 2 <= E <= 256: folds_host points to nproblems
 * structs SvmFoldWide {int n_train, n_pos, n_test, pad; int train_idx[256]; int test_idx[256];
 * unsigned char test_pos[256]} (2320 bytes; 2 <= n_train <= 256, n_test <= 256, at most 4096 problems).  Bit t % 64 of
 * bits_dev[(v*nproblems + p)*4 + t / 64] is set when sample test_idx[t] of problem p falls on the side of the first
 * class (words past the held-out samples are 0).  Same iterations and decisions as fcma_svm_cv_solve on the same
 * problems; Q is read from K_dev instead of a shared-memory copy, so it is the slower of the two at E <= 64. */
int fcma_svm_cv_solve_wide(const float *K_dev, long nv, int E, int nproblems, const void *folds_host, double C,
                           double tol, int max_iter, int shrinking, int *correct_dev, unsigned long long *bits_dev,
                           int *iters_dev, void *stream);
/* fcma_svm_cv_solve_f64 for wider problems, on fp64 kernels [nv][E][E] with 2 <= E <= 256: SvmFoldWide problems and four
 * decision words per problem, as in fcma_svm_cv_solve_wide.  Same iterations and decisions as fcma_svm_cv_solve_f64 on
 * the same problems. */
int fcma_svm_cv_solve_f64_wide(const double *K_fit_dev, const double *K_pred_dev, long nv, int E, int nproblems,
                               const void *folds_host, double C, double tol, int max_iter, int shrinking,
                               int *correct_dev, unsigned long long *bits_dev, int *iters_dev, void *stream);

/* ---- searchlight kernel matrices (MVPAVoxelSelector, mvpa_voxelselector.py:34-49 per centre) --------------------------
 * vol_dev: float32 [nx][ny][nz][E] (epochs contiguous per voxel); mask_dev: bytes [nx][ny][nz]; shape_dev: bytes
 * [2r+1]^3; centres_host: M linear voxel indices, each at least sl_rad from every face; the features of a centre are
 * the voxels of its cube where mask and shape hold, in C order.  K_fit_dev (and K_pred_dev for rbf): double [M][E][E].
 * kind 0 linear: K_fit = G = sum_f x_a x_b (K_pred_dev may be null; a separate K_pred is not written).  kind 1 rbf
 * with gamma_host[M]: K_fit = exp(-gamma ((G_aa + G_bb) - 2 G_ab)), K_pred = exp(-gamma sum_f (x_a - x_b)^2).  fp64
 * sums in cube order, no FMA contraction.  1 <= E <= 64. */
int fcma_searchlight_kernels(const float *vol_dev, long nx, long ny, long nz, int E, const unsigned char *mask_dev,
                             int sl_rad, const unsigned char *shape_dev, const long *centres_host, long M, int kind,
                             const double *gamma_host, double *K_fit_dev, double *K_pred_dev, void *stream);
/* fcma_searchlight_kernels for 1 <= E <= 256: the same arguments and outputs, computed in 64 x 64 tiles.  Every entry is
 * summed in the same order as fcma_searchlight_kernels sums it, so it depends only on the two epochs' features: the
 * entries of a subset S of the epochs equal fcma_searchlight_kernels on the volume of those epochs, bit for bit. */
int fcma_searchlight_kernels_wide(const float *vol_dev, long nx, long ny, long nz, int E, const unsigned char *mask_dev,
                                  int sl_rad, const unsigned char *shape_dev, const long *centres_host, long M, int kind,
                                  const double *gamma_host, double *K_fit_dev, double *K_pred_dev, void *stream);

/* ---- per-voxel fp64 kernels of the normalised correlation vectors (VoxelSelector with SVC(kernel='linear' | 'rbf')) ----
 * The plain pipeline of fcma_voxel_kernels (one or two masks, same operands, work buffer and passes) with a different
 * second stage.  For voxel rows [start, start+nb): z[i] = the raw correlations r[i] ([E][V2]) normalised exactly as
 * fcma_within_subject_norm does (any eps >= 1; epochs past the last whole subject keep their raw r), then, in fp64,
 * G_ab = sum_j z_aj z_bj and, for rbf, D_ab = sum_j (z_aj - z_bj)^2, in a fixed order (two runs are bit-identical).
 *   kind 0 linear: K_fit = G (K_pred_dev may be null; a separate K_pred is not written).
 *   kind 1 rbf:    K_fit = exp(-gamma ((G_aa + G_bb) - 2 G_ab)), K_fit_aa = 1; K_pred = exp(-gamma D).  gamma >= 0, finite.
 * These are the kernel values libsvm computes for SVC(kernel=...) on the float32 features z[i], so fcma_svm_cv_solve_f64
 * on them cross-validates that classifier.  Outputs double [nb][E][E]; 1 <= E <= 64. */
int fcma_voxel_feature_kernels(const void *rows_op, const void *cols_op, int precision, int E, int T, long V, long V2,
                               long start, long nb, int eps, int kind, double gamma, float *work_dev, size_t work_bytes,
                               double *K_fit_dev, double *K_pred_dev, void *stream);
/* The same for 1 <= E <= 256, same arguments and outputs: the raw block is normalised in place (within-subject z, the
 * same z as above), then one CTA per (row, upper 64 x 64 epoch tile) sums G on the fp64 tensor cores and, for rbf, D on
 * the FP64 pipe; a per-row epilogue applies the rbf forms.  D (so the rbf K_pred) is bit-identical to
 * fcma_voxel_feature_kernels' at E <= 64, G is summed in another order of its 4-column steps, every entry in the same
 * order whichever tile computes it.  Both matrices are exactly symmetric. */
int fcma_voxel_feature_kernels_wide(const void *rows_op, const void *cols_op, int precision, int E, int T, long V, long V2,
                                    long start, long nb, int eps, int kind, double gamma, float *work_dev,
                                    size_t work_bytes, double *K_fit_dev, double *K_pred_dev, void *stream);

/* ---- SVC(kernel='rbf', gamma='scale'): gamma = 1 / (F var(X_train)) per (item, fold) ---------------------------------
 * fcma_voxel_feature_kernels_wide's pipeline without the rbf epilogue: G_dev = G, D_dev = D (double [nb][E][E], the
 * entries fcma_voxel_feature_kernels_wide exponentiates), and moments_dev = double [nb][E][4]: s.hi, s.lo, q.hi, q.lo of
 * the double-double sums s_e = sum_j z_ej, q_e = sum_j z_ej^2 over the row's normalised features (fixed order).
 * 1 <= E <= 256. */
int fcma_voxel_feature_gram_wide(const void *rows_op, const void *cols_op, int precision, int E, int T, long V, long V2,
                                 long start, long nb, int eps, float *work_dev, size_t work_bytes, double *G_dev,
                                 double *D_dev, double *moments_dev, void *stream);
/* the same for searchlight centres (arguments of fcma_searchlight_kernels_wide): G and D as fcma_searchlight_kernels_wide
 * sums them, not exponentiated, and the moments of each centre's features in cube order.  1 <= E <= 256. */
int fcma_searchlight_gram_wide(const float *vol_dev, long nx, long ny, long nz, int E, const unsigned char *mask_dev,
                               int sl_rad, const unsigned char *shape_dev, const long *centres_host, long M, double *G_dev,
                               double *D_dev, double *moments_dev, void *stream);
/* gamma_dev[item][fold] = scikit-learn's gamma='scale' on the fold's training samples (train_host: bytes [nfolds][E], 1 =
 * training sample): 1 / (F * var) with var the exact variance of the n_train x F training features rounded once, 1.0 if
 * var == 0.  F = nfeat_dev[item] (int64, device) or, if nfeat_dev is null, nfeat.  flag_dev[item][fold] = 1 where
 * NumPy's two-pass variance may differ from var by more than a few ulps (mean^2 > 2^36 var; DESIGN.md §3.9). */
int fcma_fold_gammas(const double *moments_dev, long n, int E, int nfolds, const unsigned char *train_host,
                     const long *nfeat_dev, long nfeat, double *gamma_dev, unsigned char *flag_dev, void *stream);
/* rbf kernels of one fold, out of place: K_fit = exp(-g ((G_aa + G_bb) - 2 G_ab)), K_pred = exp(-g D) with
 * g = gamma_dev[item * nfolds + fold]; the operations of fcma_voxel_feature_kernels_wide's rbf epilogue. */
int fcma_rbf_fold_kernels(const double *G_dev, const double *D_dev, long n, int E, const double *gamma_dev, int nfolds,
                          int fold, double *K_fit_dev, double *K_pred_dev, void *stream);

/* ---- a12 / a15: plain NT GEMM  C[m][n] = sum_k A[m][k]*B[n][k]  (fp32 FFMA, row-major) ---------- */
int fcma_gemm_nt(const float *A_dev, const float *B_dev, float *C_dev, long M, long N, long K,
                 long lda, long ldb, long ldc, void *stream);
/* rows of X [R][D] (pitch ld) -> z-score / sqrt(D) in place, util.py:32-60; nan_to_zero as return_nans=False */
int fcma_row_normalize(float *X_dev, long R, long D, long ld, int nan_to_zero, void *stream);

/* ---- host-buffer entry points (what a cgo/ctypes binding of the reference would call) ------------ */
/* raw_host / raw2_host: E pointers to C-contiguous float32 [T_e][V] / [T_e][V2] HOST arrays
 * (raw2_host may be NULL for self-correlation); K_host: float32 [nb][E][E] HOST.  Performs H2D,
 * packing, the fused pipeline and D2H on `device`, synchronously. */
int fcma_host_voxel_kernels(const float *const *raw_host, const float *const *raw2_host,
                            const int *T_e, int E, long V, long V2, long start, long nb, int eps,
                            int precision, int normalize, int flags, int device, float *K_host);

/* the worker's whole task loop for ONE mask from host buffers (voxelselector.py:255-282 with raw_data2 None): H2D, packing,
 * fcma_voxel_kernels_sym over all V rows, D2H of K_host = float32 [V][E][E] (unshrunk), synchronously.  rows_per_pass <= 0:
 * 4096 (clamped to what fits).  Device buffers come from the device's stream-ordered pool and are reused across calls. */
int fcma_host_voxel_kernels_sym(const float *const *raw_host, const int *T_e, int E, long V, int eps,
                                int precision, int normalize, int flags, int device, long rows_per_pass,
                                float *K_host);

/* ---- inter-process peer copies over NVLink with the copy engines (one process per GPU of a box) ------------------
 * Replaces the per-epoch comm.bcast loop of prepare_fcma_data (preprocessing.py:211-223) without occupying SMs:
 * every rank uploads ITS share of the epochs over its own PCIe link, exports the destination buffer as a CUDA IPC
 * handle (64 bytes + the offset of dev_ptr inside its allocation), the peers map it and copy their shares into it.
 * The library keeps no state; mappings are closed by the caller. */
int fcma_ipc_get_handle(const void *dev_ptr, void *handle64, size_t *offset);
int fcma_ipc_open_handle(const void *handle64, void **base_ptr);
int fcma_ipc_close_handle(void *base_ptr);
int fcma_peer_copy_async(void *dst_dev, const void *src_dev, size_t bytes, void *stream);

/* in-place host variants of the reference's native functions */
int fcma_host_within_subject_norm(float *corr_host, long n0, int E, long n2, int eps, int device);

/* per-kernel timing of the fused pipelines (CUDA events on the launch stream; synchronises each pass):
 * enable(1) resets the accumulators; read() returns the number of passes and the summed milliseconds of
 * the correlation GEMM (+ diagonal fix-up) and of the normalise+SYRK kernel */
void fcma_timing_enable(int on);
long fcma_timing_read(double *gemm_ms, double *syrk_ms);
/* same with the normalise+SYRK time split: syrk_ms = first launch of a pass (rows of the block), syrk2_ms = second
 * launch of a symmetric pass (column-direction pass, or the row pass over the transposed block) */
long fcma_timing_read3(double *gemm_ms, double *syrk_ms, double *syrk2_ms);

/* number of kernel launches issued by this library in the calling process (for bench accounting) */
long fcma_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FCMA_B200_H */
