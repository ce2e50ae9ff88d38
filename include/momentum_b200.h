/*
 * momentum_b200 — C-ABI of the H100-native (sm_90a) batched Gauss-Newton IK path.
 *
 * This is the drop-in boundary for ONE hot path of facebookresearch/momentum: the per-iteration
 * FK sweep -> residual/Jacobian (Position / Orientation / State / Limit) -> JtJ, Jtr -> damped
 * Cholesky -> parameter update, for a BATCH of independent IK instances that share one rig and one
 * constraint topology (the body of the dispenso::parallel_for at
 * pymomentum/tensor_ik/tensor_ik.cpp:127-177). Every entry point below names the reference
 * interface it stands in for (paths relative to the reference's momentum/ directory).
 *
 * Conventions
 *  - plain C types only; no C++/torch types cross this boundary.
 *  - every function returns MB2_OK (0) or an error code; mb2_last_error() gives the message of the
 *    last failure on the calling thread (reference: MT_CHECK/MT_THROW -> std::runtime_error,
 *    common/checks.h:36, common/exception.h:31; adapters rethrow).
 *  - host pointers unless the name says _device. Host inputs are copied during the call and never
 *    retained (reference ownership: the solver holds non-owning pointers, solver/solver.h:106).
 *  - handles are not thread-safe; one handle = one CUDA stream (reference: one solver + function per
 *    thread, tensor_ik.cpp:127-162; mutable scratch in skeleton_solver_function.h:89).
 *  - quaternions are (x, y, z, w) like Eigen::Quaternion::coeffs().
 *  - batched arrays are instance-major: [B][...].
 *  - there is no CPU fallback: every compute entry point fails with MB2_ERR_CUDA when no sm_90
 *    device is usable.
 */
#ifndef MOMENTUM_B200_H_
#define MOMENTUM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB2_PARAMETERS_PER_JOINT 7   /* character/types.h:21 kParametersPerJoint */
#define MB2_MAX_MODEL_PARAMETERS 2048 /* math/types.h:426-429 ParameterSet = std::bitset<2048> */
#define MB2_PARAMETER_SET_WORDS 32   /* 2048 / 64 */

typedef enum mb2_status {
  MB2_OK = 0,
  MB2_ERR_INVALID_ARGUMENT = 1, /* MT_CHECK failure in the reference */
  MB2_ERR_CUDA = 2,             /* CUDA runtime error / no usable device (no CPU fallback) */
  MB2_ERR_UNSUPPORTED = 3
} mb2_status;

/* Per-instance result status of a batched solve (reference: NaN/Inf guard of the batched caller,
 * tensor_ik.cpp:168-173; LLT info is ignored by the dense solver, gauss_newton_solver.cpp:251). */
typedef enum mb2_instance_status {
  MB2_INSTANCE_OK = 0,
  MB2_INSTANCE_CHOLESKY_BREAKDOWN = 1, /* a non-positive pivot was met (Eigen: NumericalIssue) */
  MB2_INSTANCE_NON_FINITE = 2          /* parameters became NaN/Inf */
} mb2_instance_status;

/* character/parameter_limits.h:20-33 LimitType */
typedef enum mb2_limit_type {
  MB2_LIMIT_MINMAX = 0,
  MB2_LIMIT_MINMAX_JOINT = 1,
  MB2_LIMIT_MINMAX_JOINT_PASSIVE = 2,
  MB2_LIMIT_LINEAR = 3,
  MB2_LIMIT_LINEAR_JOINT = 4,
  MB2_LIMIT_ELLIPSOID = 5,
  MB2_LIMIT_HALFPLANE = 6
} mb2_limit_type;

/* character/parameter_limits.h:117-127 ParameterLimit, flattened.
 *  MinMax:      i[0]=parameterIndex, f[0..1]=limits
 *  MinMaxJoint: i[0]=jointIndex, i[1]=jointParameter, f[0..1]=limits
 *  Linear:      i[0]=referenceIndex, i[1]=targetIndex, f[0]=scale, f[1]=offset, f[2]=rangeMin, f[3]=rangeMax
 *  LinearJoint: i[0..1]=reference joint/param, i[2..3]=target joint/param, f[0..3] as Linear
 *  HalfPlane:   i[0]=param1, i[1]=param2, f[0..1]=normal, f[2]=offset
 *  Ellipsoid:   i[0]=ellipsoidParent, i[1]=parent, f[0..11]=ellipsoid 3x4 row-major, f[12..23]=ellipsoidInv, f[24..26]=offset */
typedef struct mb2_parameter_limit {
  int32_t type;
  float weight;
  int32_t i[4];
  float f[27];
} mb2_parameter_limit;

/* state_error_function.h:17-32 RotationErrorType */
typedef enum mb2_rotation_error_type {
  MB2_ROTATION_MATRIX_DIFFERENCE = 0,
  MB2_QUATERNION_LOG_MAP = 1
} mb2_rotation_error_type;

/* How JtJ is formed on the device (extension; the reference always uses Eigen fp32/fp64 GEMM). */
typedef enum mb2_jtj_mode {
  MB2_JTJ_AUTO = 0,      /* tile-sparse Gram (mma.sync, three-term TF32 split: fp32-class, not bit-exact fp32) with the tile-scheduled Cholesky; else wgmma 3xTF32 where the shape allows, else FP32 SIMT */
  MB2_JTJ_FP32_SIMT = 1, /* CUDA-core fp32 (validation path) */
  MB2_JTJ_TF32X3 = 2,    /* wgmma tf32, 3-term split, fp32 accumulate in registers (fp32-class accuracy); up to 511 Jacobian columns */
  MB2_JTJ_TF32 = 3,      /* wgmma tf32 single pass (~1e-3 relative; changes the GN path, not the fixed point) */
  MB2_JTJ_SPARSE_TILES = 4 /* tensor cores (mma.sync m16n8k8, hi*hi + hi*lo + lo*hi TF32 split, the lo*lo term is dropped: ~2^-21 relative) over the non-zero
                              strips of J only, straight into the Cholesky tile layout (tile-scheduled Cholesky only) */
} mb2_jtj_mode;

/* How (JtJ + lambda I) delta = Jtr is solved on the device (extension; the reference always runs a dense
 * Eigen::LLT, gauss_newton_solver.cpp:251). All modes solve the same system; they differ in elimination
 * order (rounding) and in what happens on a non-positive pivot: the dense Eigen-structured kernel
 * reproduces Eigen's early exit, the tile schedules substitute the damping for the pivot; both flag the
 * instance MB2_INSTANCE_CHOLESKY_BREAKDOWN. */
typedef enum mb2_cholesky_mode {
  MB2_CHOLESKY_AUTO = 0,            /* tile schedule on the sparsity pattern for >= 48 unknowns, else dense Eigen-structured */
  MB2_CHOLESKY_DENSE_EIGEN = 1,     /* blocked LLT with Eigen's block structure and failure semantics */
  MB2_CHOLESKY_TILES_DENSE = 2,     /* level-scheduled 16x16 tiles, every tile present */
  MB2_CHOLESKY_TILES_SPARSE = 3     /* level-scheduled tiles over the kinematic-tree sparsity of JtJ (min-degree order) */
} mb2_cholesky_mode;

/* Which kernels run one Gauss-Newton iteration on the tile path (extension; every mode solves the same system with the same device
 * functions, results agree to float rounding).
 *   GRAM_CHOLESKY  two launches per iteration: FK / residual / Jacobian strips, then ONE kernel that forms the stored tiles of
 *                  J^T J + lambda I from the strips on the tensor cores (a tile that would overwrite strips still being read waits in
 *                  an L2-resident scratch slot), writes them over the dead strips in shared memory and runs the tile Cholesky + update on them.
 *   OFF            three launches per iteration (sweep, tile-sparse Gram to HBM, tile Cholesky).
 *   PERSISTENT     ONE launch per solve: groups of 256 threads keep an instance in shared memory for all of its iterations (FK sweep
 *                  included) and stop it on the device; no host round trip, no HBM traffic beyond theta / targets / results. Needs no
 *                  line search and a plan whose tiles fit in shared memory next to the staged tables. At most three instances per SM
 *                  are in flight, so AUTO takes it only for a batch of one wave of instance groups. */
typedef enum mb2_fused_mode {
  MB2_FUSED_AUTO = 0,          /* PERSISTENT when the batch is a single wave of instance groups (<= 3 per SM), else GRAM_CHOLESKY when strips / tiles fit in
                                  shared memory, else OFF */
  MB2_FUSED_OFF = 1,
  MB2_FUSED_PERSISTENT = 2,    /* or MB2_ERR_UNSUPPORTED */
  MB2_FUSED_GRAM_CHOLESKY = 3  /* or MB2_ERR_UNSUPPORTED */
} mb2_fused_mode;

/* How the Gauss-Newton step is computed from the Jacobian. CHOLESKY = GaussNewtonSolverT / SubsetGaussNewtonSolverT (normal equations,
 * Eigen::LLT; gauss_newton_solver.cpp:248-251). QR = GaussNewtonSolverQRT (character_solver/gauss_newton_solver_qr.cpp:50-150): an online
 * Householder QR of [sqrt(lambda) I; J] (math/online_householder_qr.cpp), the default solver of pymomentum's solve_ik and of the marker
 * tracker; same step up to rounding without squaring the condition number; its line search is the c1 = 1e-4 / g.delta rule (:116-143). */
typedef enum mb2_linear_solver {
  MB2_LINEAR_SOLVER_CHOLESKY = 0,
  MB2_LINEAR_SOLVER_QR = 1,
  /* TrustRegionQRT (character_solver/trust_region_qr.cpp:52-270; LinearSolverType::TrustRegionQR of pymomentum's solve_ik): QR of the
   * Jacobian, a Newton search for the damping that keeps the step inside the trust region, rho-driven radius, steps with rho <= 0 rejected.
   * regularization, do_line_search and use_block_jtj do not apply (the reference's class takes plain SolverOptions + the radius). */
  MB2_LINEAR_SOLVER_TRUST_REGION_QR = 2
} mb2_linear_solver;

/* solver/solver.h:19-34 SolverOptions + solver/gauss_newton_solver.h:17-59 GaussNewtonSolverOptions,
 * field for field, plus device extensions at the end. */
typedef struct mb2_gauss_newton_options {
  uint64_t min_iterations;        /* SolverOptions::minIterations = 1 */
  uint64_t max_iterations;        /* SolverOptions::maxIterations = 2 */
  float threshold;                /* SolverOptions::threshold = 1.0f */
  int32_t verbose;                /* SolverOptions::verbose */
  float regularization;           /* GaussNewtonSolverBaseOptions::regularization = 0.05f */
  int32_t do_line_search;         /* ::doLineSearch = false */
  int32_t use_block_jtj;          /* ::useBlockJtJ = false (same normal equations either way) */
  uint64_t target_rows_per_chunk; /* ::targetRowsPerChunk = SIZE_MAX (accepted, no effect on results) */
  int32_t subset_line_search;     /* 1 = SubsetGaussNewtonSolverT line search (c1=1e-4, g.delta), subset_gauss_newton_solver.cpp:119-141 */
  int32_t jtj_mode;               /* mb2_jtj_mode */
  int32_t store_error_history;    /* keep per-iteration error per instance (solver.h:90 getErrorHistory) */
  int32_t cholesky_mode;          /* mb2_cholesky_mode */
  int32_t fused_mode;             /* mb2_fused_mode */
  int32_t linear_solver;          /* mb2_linear_solver */
  float trust_region_radius;      /* TrustRegionQROptions::trustRegionRadius_ = 1.0f (trust_region_qr.h:23); MB2_LINEAR_SOLVER_TRUST_REGION_QR only */
} mb2_gauss_newton_options;

typedef struct mb2_character mb2_character;             /* Skeleton + ParameterTransform + ParameterLimits on device */
typedef struct mb2_solver_function mb2_solver_function; /* batch of B SkeletonSolverFunctionT<float> */
typedef struct mb2_solver mb2_solver;                   /* batch of B GaussNewtonSolverT<float> */

const char* mb2_last_error(void);
/* number of usable sm_90 devices (0 => every compute call fails with MB2_ERR_CUDA) */
int mb2_device_count(void);
void mb2_default_gauss_newton_options(mb2_gauss_newton_options* opt);

/* ---- Character: Skeleton (character/skeleton.h:22-77, joint.h:18-76) + ParameterTransform
 * (character/parameter_transform.h:62-184; CSR rows = 7*num_joints) ------------------------------- */
int mb2_character_create(int device, int32_t num_joints, const int32_t* parents /*[J], -1 root*/,
                         const float* translation_offsets /*[J*3]*/, const float* pre_rotations /*[J*4] xyzw*/,
                         int32_t num_model_parameters, const int32_t* transform_outer /*[7J+1]*/,
                         const int32_t* transform_inner /*[nnz]*/, const float* transform_values /*[nnz]*/,
                         const float* transform_offsets /*[7J]*/, mb2_character** out);
/* ParameterLimits consumed by LimitErrorFunctionT (character/parameter_limits.h:129) */
int mb2_character_set_parameter_limits(mb2_character* c, int32_t count, const mb2_parameter_limit* limits);
void mb2_character_destroy(mb2_character* c);

/* ---- SkeletonSolverFunctionT<float> x B (character_solver/skeleton_solver_function.h:21-95) ---- */
int mb2_solver_function_create(const mb2_character* c, int32_t batch, mb2_solver_function** out);
void mb2_solver_function_destroy(mb2_solver_function* f);
int32_t mb2_solver_function_num_parameters(const mb2_solver_function* f);    /* getNumParameters */
int32_t mb2_solver_function_actual_parameters(const mb2_solver_function* f); /* getActualParameters */
int32_t mb2_solver_function_batch(const mb2_solver_function* f);
/* getJacobianBlockSize summed and padded to 8 (solver_function.cpp:33-38) */
int32_t mb2_solver_function_jacobian_rows(const mb2_solver_function* f);
/* row stride (leading dimension) of device Jacobian columns */
int32_t mb2_solver_function_jacobian_stride(const mb2_solver_function* f);

/* addErrorFunction(PositionErrorFunctionT) — position_error_function.h:16-73. Constraint topology
 * (parent, offset, weight) is shared by the batch; targets are per instance. Returns block index. */
int mb2_add_position_error_function(mb2_solver_function* f, float weight, float loss_alpha, float loss_c,
                                    int32_t num_constraints, const int32_t* parents, const float* offsets /*[nc*3]*/,
                                    const float* weights /*[nc]*/, int32_t* out_index);
/* Same, with the constraint OFFSETS per instance as well (the reference builds its error functions per batch element,
 * pymomentum/tensor_ik/tensor_ik.cpp:136-140: offsets and targets may differ from element to element; the parent joints fix the
 * sparsity pattern and stay shared). Per-instance record (mb2_set_targets): [B][nc*6] = target xyz, offset xyz per constraint. */
int mb2_add_position_error_function_instanced(mb2_solver_function* f, float weight, float loss_alpha, float loss_c, int32_t num_constraints,
                                              const int32_t* parents, const float* weights /*[nc]*/, int32_t* out_index);
/* Orientation (matrix difference, rot_diff = 0, or rot-diff) with the constraint OFFSETS per instance, like the Position one above.
 * Per-instance record (mb2_set_targets[_device]): [B][nc*8] = target xyzw, offset xyzw per constraint; both are normalised on upload. */
int mb2_add_orientation_error_function_instanced(mb2_solver_function* f, float weight, float loss_alpha, float loss_c, int32_t rot_diff,
                                                 int32_t num_constraints, const int32_t* parents, const float* weights /*[nc]*/, int32_t* out_index);
/* addErrorFunction(PlaneErrorFunctionT) — plane_error_function.h:20-101, .cpp:49-70: signed distance of T_parent * offset to the plane
 * (normal, d), one residual row per constraint; above != 0 is the half-plane mode (only val < 0 is penalised). Per-instance targets
 * (mb2_set_targets): [B][nc*4] = normal xyz (normalised as in PlaneDataT's ctor), d. kLegacyWeight = 1e-4 (.h:83). */
int mb2_add_plane_error_function(mb2_solver_function* f, float weight, float loss_alpha, float loss_c, int32_t above,
                                 int32_t num_constraints, const int32_t* parents, const float* offsets /*[nc*3]*/,
                                 const float* weights /*[nc]*/, int32_t* out_index);
/* addErrorFunction(ModelParametersErrorFunctionT) — model_parameters_error_function.h/.cpp: row sqrt(weight * kMotionWeight) * w_i *
 * (theta_i - target_i) for every enabled parameter with target weight w_i > 0 (kMotionWeight = 1e-1, .h:61). Per-instance targets
 * (mb2_set_targets): [B][numParams] target parameters; target_weights [numParams] is shared by the batch. */
int mb2_add_model_parameters_error_function(mb2_solver_function* f, float weight, const float* target_weights /*[numParams]*/,
                                            int32_t* out_index);
/* addErrorFunction(OrientationErrorFunctionT / OrientationRotDiffErrorFunctionT) —
 * orientation_error_function.h:16-108; offsets are normalised as in OrientationDataT's ctor. */
int mb2_add_orientation_error_function(mb2_solver_function* f, float weight, float loss_alpha, float loss_c,
                                       int32_t rot_diff, int32_t num_constraints, const int32_t* parents,
                                       const float* offsets /*[nc*4]*/, const float* weights /*[nc]*/, int32_t* out_index);
/* addErrorFunction(StateErrorFunctionT) — state_error_function.h:35-117 (setWeights, setTargetWeights) */
int mb2_add_state_error_function(mb2_solver_function* f, float weight, int32_t rotation_error_type, float pos_wgt,
                                 float rot_wgt, const float* target_position_weights /*[J]*/,
                                 const float* target_rotation_weights /*[J]*/, int32_t* out_index);
/* addErrorFunction(LimitErrorFunctionT) over the character's limits — limit_error_function.h:25-119 */
int mb2_add_limit_error_function(mb2_solver_function* f, float weight, float loss_alpha, float loss_c, int32_t* out_index);
/* SkeletonErrorFunctionT::setWeight (skeleton_error_function.h:45-47) */
int mb2_set_error_function_weight(mb2_solver_function* f, int32_t index, float weight);
/* Per-instance targets: Position [B*nc*3] (setConstraints targets), Orientation [B*nc*4] xyzw
 * (normalised on upload), State [B*J*8] = (t, q xyzw, s) (setTargetState). */
int mb2_set_targets(mb2_solver_function* f, int32_t index, const float* targets);
int mb2_set_targets_device(mb2_solver_function* f, int32_t index, const float* targets_device, void* cuda_stream);
/* Optional per-instance constraint weights [B*nc] for a Position/Orientation block (ConstraintData::weight) */
int mb2_set_constraint_weights(mb2_solver_function* f, int32_t index, const float* weights, int32_t per_instance);
/* the same from device memory, [B][nc] contiguous, on `cuda_stream` (NULL = handle stream) */
int mb2_set_constraint_weights_device(mb2_solver_function* f, int32_t index, const float* weights_device, void* cuda_stream);
/* SolverFunctionT::setEnabledParameters(ParameterSet) — skeleton_solver_function.cpp:45-61 */
int mb2_solver_function_set_enabled_parameters(mb2_solver_function* f, const uint64_t bits[MB2_PARAMETER_SET_WORDS]);

/* SolverFunctionT::getError — skeleton_solver_function.cpp:64-83 (value rounded through float). */
int mb2_solver_function_get_error(mb2_solver_function* f, const float* parameters /*[B*n]*/, double* errors /*[B]*/);
/* SolverFunctionT::getJacobian — solver_function.cpp:22-71. jacobian [B][n][rows] (column-major per
 * instance, rows = mb2_solver_function_jacobian_rows), residual [B][rows]. */
int mb2_solver_function_get_jacobian(mb2_solver_function* f, const float* parameters, float* jacobian, float* residual,
                                     double* errors, int32_t* actual_rows);
/* getJacobian with parameters and result on the device (no copy): *jacobian_device points at the handle's Jacobian buffer,
 * [B][n + 1][ld] floats, column c of instance b at ((b * (n + 1)) + c) * ld, column n = residual; rows beyond
 * mb2_solver_function_jacobian_rows are zero. Valid until the next call on the handle. */
int mb2_solver_function_get_jacobian_device(mb2_solver_function* f, const float* parameters_device, const float** jacobian_device, int32_t* ld, void* cuda_stream);
/* SolverFunctionT::getJtJR — solver_function.cpp:74-121. jtj [B][ap][ap] (lower triangle valid,
 * ap = actual parameters), jtr [B][ap]. */
int mb2_solver_function_get_jtjr(mb2_solver_function* f, const float* parameters, int32_t jtj_mode, float* jtj, float* jtr,
                                 double* errors);
/* Skeleton state after initializeJacobianComputation (skeleton_state.cpp:87-121): [B][J][8] (t,q,s) */
int mb2_solver_function_get_skeleton_state(mb2_solver_function* f, const float* parameters, float* state);

/* Differentiable forward kinematics on the character alone, device memory in and out, on `cuda_stream` (NULL = the legacy default
 * stream), asynchronous. batch == 0 is a no-op. A null pointer (batch > 0), batch < 0, or a pointer that is not device memory on the
 * character's device is MB2_ERR_INVALID_ARGUMENT.
 * pymomentum model_parameters_to_skeleton_state (tensor_skeleton_state.cpp:500-502, :213-270): [B][n] -> [B][J][8] (t, q xyzw, s) */
int mb2_character_skeleton_state_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                        float* skeleton_state_device, void* cuda_stream);
/* its backward (computeSkelStateBackward, :62-134, then the ParameterTransform transposed): dLoss/dtheta [B][n], overwritten */
int mb2_character_skeleton_state_backward_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                 const float* grad_skeleton_state_device, float* grad_model_parameters_device,
                                                 void* cuda_stream);

/* The skeleton-state family on the character alone, both directions, with the argument rules of mb2_character_skeleton_state_device.
 * Joint parameters are [B][7 J] (joint j's seven values t xyz, rx ry rz, log2 scale at 7 j), states [B][J][8] (t, q xyzw, s). Every
 * backward overwrites dLoss / d its forward's input from dLoss / d its forward's output.
 * pymomentum apply_parameter_transform (diff_transform_pybind.cpp:27, tensor_parameter_transform.cpp:195-209): [B][n] -> P theta + o
 * [B][7 J]; its backward is P^T, so it reads no input (model_parameters_device may be null there). */
int mb2_character_apply_parameter_transform_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                   float* joint_parameters_device, void* cuda_stream);
int mb2_character_apply_parameter_transform_backward_device(const mb2_character* c, int32_t batch, const float* grad_joint_parameters_device,
                                                            float* grad_model_parameters_device, void* cuda_stream);
/* pymomentum apply_inverse_parameter_transform (diff_transform_pybind.cpp:44-59, tensor_parameter_transform.cpp:378-466):
 * [B][7 J] -> theta = W (jp - o) [B][n], the offsets subtracted first, with W = P^+ the Moore-Penrose pseudo-inverse of
 * InverseParameterTransform (inverse_parameter_transform.cpp:18-38) under its rule of utility.cpp:423-435: a singular value > 1e-6
 * (absolute) is inverted, any other is 0. W is built once per character, in float64 per connected component of P's sparsity pattern, and
 * rounded to float entry by entry. The `offsets` half of InverseParameterTransform::apply is not returned. Its backward is W^T, so it
 * reads no input. */
int mb2_character_apply_inverse_parameter_transform_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                           float* model_parameters_device, void* cuda_stream);
int mb2_character_apply_inverse_parameter_transform_backward_device(const mb2_character* c, int32_t batch, const float* grad_model_parameters_device,
                                                                    float* grad_joint_parameters_device, void* cuda_stream);
/* pymomentum joint_parameters_to_skeleton_state (tensor_skeleton_state.cpp:203-343, :488-491): the forward kinematics of
 * mb2_character_skeleton_state_device from joint parameters [B][7 J] -> [B][J][8] */
int mb2_character_joint_parameters_to_skeleton_state_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                            float* skeleton_state_device, void* cuda_stream);
int mb2_character_joint_parameters_to_skeleton_state_backward_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                                     const float* grad_skeleton_state_device, float* grad_joint_parameters_device,
                                                                     void* cuda_stream);
/* pymomentum joint_parameters_to_local_skeleton_state (:346-484, backward computeLocalSkelStateBackward :139, :493-498): each joint's
 * transform to its parent, t = offset + p[0:3], q = preRot Rz(p5) Ry(p4) Rx(p3), s = 2^p6: [B][7 J] -> [B][J][8] */
int mb2_character_joint_parameters_to_local_skeleton_state_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                                  float* local_skeleton_state_device, void* cuda_stream);
int mb2_character_joint_parameters_to_local_skeleton_state_backward_device(const mb2_character* c, int32_t batch,
                                                                           const float* joint_parameters_device,
                                                                           const float* grad_local_skeleton_state_device,
                                                                           float* grad_joint_parameters_device, void* cuda_stream);
/* pymomentum local_skeleton_state_to_joint_parameters (:611-648): t - offset, the XYZ Euler angles of inv(preRot) q (the asin argument
 * clamped to [-1, 1], where its derivative is 0), log2 s: [B][J][8] -> [B][J][7] */
int mb2_character_local_skeleton_state_to_joint_parameters_device(const mb2_character* c, int32_t batch, const float* local_skeleton_state_device,
                                                                  float* joint_parameters_device, void* cuda_stream);
int mb2_character_local_skeleton_state_to_joint_parameters_backward_device(const mb2_character* c, int32_t batch,
                                                                           const float* local_skeleton_state_device,
                                                                           const float* grad_joint_parameters_device,
                                                                           float* grad_local_skeleton_state_device, void* cuda_stream);
/* pymomentum skeleton_state_to_joint_parameters (:650-668): the local states inv(X_parent) X_j (identity above a root), then the rule
 * above: [B][J][8] -> [B][J][7] */
int mb2_character_skeleton_state_to_joint_parameters_device(const mb2_character* c, int32_t batch, const float* skeleton_state_device,
                                                            float* joint_parameters_device, void* cuda_stream);
int mb2_character_skeleton_state_to_joint_parameters_backward_device(const mb2_character* c, int32_t batch, const float* skeleton_state_device,
                                                                     const float* grad_joint_parameters_device, float* grad_skeleton_state_device,
                                                                     void* cuda_stream);

/* pymomentum model_parameters_to_positions / joint_parameters_to_positions (geometry_pybind.cpp:1131-1171,
 * tensor_joint_parameters_to_positions.cpp:33-52, :320-327): the world positions of num_points points fixed in joints' frames,
 * p_i = t_a + rot(q_a, s_a offsets_i) with (t_a, q_a, s_a) the world state of joint a = parents[i] (the position constraint's point).
 * Parameters [B][n] (model) or [B][7 J] (joint), parents [num_points] in HOST memory, offsets [num_points][3] shared by the batch
 * (offsets_batched == 0) or [B][num_points][3], positions [B][num_points][3]. The argument rules of mb2_character_skeleton_state_device;
 * besides, num_points < 0 or a parent outside [0, J) (checkValidBoneIndex) is MB2_ERR_INVALID_ARGUMENT. num_points == 0 is valid: the
 * point arrays may then be NULL. The call uploads the points grouped by joint into stream-ordered scratch (cudaMallocAsync). */
int mb2_character_model_parameters_to_positions_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                       int32_t num_points, const int32_t* parents, const float* offsets_device,
                                                       int32_t offsets_batched, float* positions_device, void* cuda_stream);
int mb2_character_joint_parameters_to_positions_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                       int32_t num_points, const int32_t* parents, const float* offsets_device,
                                                       int32_t offsets_batched, float* positions_device, void* cuda_stream);
/* their backward (d_jointParametersToPositions, :54-119; the model variant then the ParameterTransform transposed) from dLoss/d positions
 * [B][num_points][3]: grad_params [B][n] ([B][7 J]) and grad_offsets in the offset layout ([num_points][3] = the batch sum when shared),
 * both overwritten. Either output may be NULL, not both. Same rules as the forward. A shared-offset gradient takes stream-ordered scratch
 * from the device's default memory pool: at most 256 MiB of per-instance rows and 128 x num_points x 3 floats of chunk sums. */
int mb2_character_model_parameters_to_positions_backward_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                                int32_t num_points, const int32_t* parents, const float* offsets_device,
                                                                int32_t offsets_batched, const float* grad_positions_device,
                                                                float* grad_model_parameters_device, float* grad_offsets_device, void* cuda_stream);
int mb2_character_joint_parameters_to_positions_backward_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                                int32_t num_points, const int32_t* parents, const float* offsets_device,
                                                                int32_t offsets_batched, const float* grad_positions_device,
                                                                float* grad_joint_parameters_device, float* grad_offsets_device, void* cuda_stream);

/* Linear-blend skinning of the character (SkinWeights, skin_weights.h:19-40, and Character::inverseBindPose), host arrays, replacing
 * any earlier skinning: rest_vertices [V][3], skin_index / skin_weight [V][8] (a vertex's influences end at its first zero weight,
 * linear_skinning.cpp:76-80; the slots after it are ignored whatever they hold), inverse_bind_pose [J][12] (the row-major top 3x4 of
 * Affine3f::matrix()). An active slot's index outside [0, J) or non-finite weight, a non-finite vertex or inverse bind pose, or V < 1 is
 * MB2_ERR_INVALID_ARGUMENT, and leaves any earlier skinning in place (as does a failed upload). The new tables go to fresh device
 * buffers and the call synchronises the device before it frees the old ones, so skinning work already enqueued on any stream finishes
 * with the tables it was enqueued with; the call must not run concurrently with another call on the same character from another host
 * thread. mb2_character_clone copies the skinning. */
int mb2_character_set_skinning(mb2_character* c, int32_t num_vertices, const float* rest_vertices, const int32_t* skin_index,
                               const float* skin_weight, const float* inverse_bind_pose);
/* V of the skinning, 0 when the character has none */
int32_t mb2_character_num_vertices(const mb2_character* c);
/* pymomentum Character.skin_points (pymomentum/torch/character.py:1050-1068; applySSD, linear_skinning.cpp:40-102, with
 * computeSkinningTransforms, :22-37, and q normalised as skel_state_backend.py:435-512 does): skel_state [B][J][8] -> points [B][V][3].
 * rest_points NULL = the character's rest mesh, else [V][3] shared by the batch (rest_points_batched == 0) or [B][V][3] (== 1).
 * Device memory on `cuda_stream`, asynchronous; batch == 0 is a no-op. No skinning, a null required pointer, batch < 0 or a pointer
 * that is not device memory on the character's device is MB2_ERR_INVALID_ARGUMENT. */
int mb2_character_skin_points_device(const mb2_character* c, int32_t batch, const float* skel_state_device, const float* rest_points_device,
                                     int32_t rest_points_batched, float* points_device, void* cuda_stream);
/* its backward (SkinPointsFunction::backward, tensor_skinning.cpp:171-330) from dLoss/d points [B][V][3]: grad_skel_state [B][J][8],
 * grad_rest_points in the rest-point layout ([V][3] = the batch sum when shared, :320-322), both overwritten, a NULL output is skipped.
 * grad_rest_points must be NULL when the rest mesh is skinned. Same rules as the forward. The call takes stream-ordered scratch from
 * the device's default memory pool (cudaMallocAsync / cudaFreeAsync on `cuda_stream`): at most 256 MiB for the skel-state gradient and
 * 128 x V x 3 floats for a shared rest-point gradient. A framework's own caching allocator does not see it. */
int mb2_character_skin_points_backward_device(const mb2_character* c, int32_t batch, const float* skel_state_device, const float* rest_points_device,
                                              int32_t rest_points_batched, const float* grad_points_device, float* grad_skel_state_device,
                                              float* grad_rest_points_device, void* cuda_stream);

/* The identity blend shape of the character (BlendShape, blend_shape.h), host arrays, replacing any earlier one: base_shape [V][3] and
 * shape_vectors [K][V][3] (shapeVectors_, 3V x K column-major, as it lies in memory). K < 1, V < 1, a null array or a non-finite value is
 * MB2_ERR_INVALID_ARGUMENT and leaves any earlier blend shape in place (as does a failed upload). Fresh device buffers and a device
 * synchronisation before the old ones are freed, as mb2_character_set_skinning. V is checked against the skinning's when skinning.
 * mb2_character_clone copies the blend shape. */
int mb2_character_set_blend_shape(mb2_character* c, int32_t num_shapes, int32_t num_vertices, const float* base_shape, const float* shape_vectors);
/* K of the blend shape, 0 when the character has none */
int32_t mb2_character_num_blend_shapes(const mb2_character* c);
/* skinWithBlendShapes (blend_shape_skinning.cpp:50-140): the rest point of every vertex is base_shape + the first num_weights shape
 * vectors weighted by blend_weights [B][num_weights] (1 <= num_weights <= K, computeDeltas' leftCols, blend_shape_base.cpp:18-24), then
 * skinned as mb2_character_skin_points_device skins: skel_state [B][J][8] -> points [B][V][3]. No shaped rest mesh is written. Device
 * memory on `cuda_stream`, asynchronous; batch == 0 is a no-op. No skinning or no blend shape, a blend shape whose V differs from the
 * skinning's, num_weights out of range or so large that the weights of a 4-instance tile and the J transforms do not fit in shared
 * memory, a null required pointer, batch < 0 or a pointer that is not device memory on the character's
 * device is MB2_ERR_INVALID_ARGUMENT. */
int mb2_character_skin_with_blend_shapes_device(const mb2_character* c, int32_t batch, const float* skel_state_device, const float* blend_weights_device,
                                                int32_t num_weights, float* points_device, void* cuda_stream);
/* its backward from dLoss/d points [B][V][3]: grad_skel_state [B][J][8] and grad_blend_weights [B][num_weights], both overwritten, a NULL
 * output is skipped. Same rules as the forward. The call takes stream-ordered scratch from the device's default memory pool
 * (cudaMallocAsync / cudaFreeAsync on `cuda_stream`): at most 256 MiB of shaped rest points plus the skin-points backward's scratch for
 * the skel-state gradient, and at most 256 MiB of partial sums for the weight gradient. */
int mb2_character_skin_with_blend_shapes_backward_device(const mb2_character* c, int32_t batch, const float* skel_state_device,
                                                         const float* blend_weights_device, int32_t num_weights, const float* grad_points_device,
                                                         float* grad_skel_state_device, float* grad_blend_weights_device, void* cuda_stream);

/* The triangles of the character's mesh (Mesh::faces, mesh.h), a host array faces [F][3] of vertex indices in [0, num_vertices),
 * replacing any earlier ones; num_faces == 0 with a null array removes them. num_vertices < 1, num_faces < 0, 3 x num_faces beyond
 * int32, a null array with num_faces > 0 or an index out of range is MB2_ERR_INVALID_ARGUMENT and leaves the earlier faces in place
 * (as does a failed upload). Degenerate faces and faces that repeat an index are accepted. The vertex -> corner table the kernels
 * gather from is built here, once. Fresh device buffers and a device synchronisation before the old ones are freed, as
 * mb2_character_set_skinning. mb2_character_clone copies the faces. */
int mb2_character_set_mesh_faces(mb2_character* c, int32_t num_vertices, int32_t num_faces, const int32_t* faces);
/* F of the mesh faces, 0 when the character has none */
int32_t mb2_character_num_faces(const mb2_character* c);
/* Area-weighted vertex normals (pymomentum compute_vertex_normals, tensor_skinning.cpp:354-383): n_v = the sum of (x1 - x0) x (x2 - x0)
 * over every corner of every face that is vertex v, faces ascending, corners in order (the sum of MeshT::updateNormals, mesh.cpp:17-51),
 * and normals = n_v / max(|n_v|, 1e-12) (torch.nn.functional.normalize): an isolated vertex gives 0. positions [B][V][3] -> normals
 * [B][V][3], V = the faces' num_vertices. Non-finite positions propagate (updateNormals' skip of NaN faces is not copied). Device
 * memory on `cuda_stream`, asynchronous; batch == 0 is a no-op. No faces, a null pointer, batch < 0 or a pointer that is not device
 * memory on the character's device is MB2_ERR_INVALID_ARGUMENT. No atomics: an instance gets the same bits alone as in any batch. */
int mb2_character_vertex_normals_device(const mb2_character* c, int32_t batch, const float* positions_device, float* normals_device, void* cuda_stream);
/* its backward from dLoss/d normals [B][V][3]: grad_positions [B][V][3], overwritten, the exact derivative including the clamp branch.
 * Same rules as the forward. The call takes stream-ordered scratch from the device's default memory pool (cudaMallocAsync /
 * cudaFreeAsync on `cuda_stream`): [slice][V][3] floats of at most 256 MiB, the instances processed in slices. */
int mb2_character_vertex_normals_backward_device(const mb2_character* c, int32_t batch, const float* positions_device, const float* grad_normals_device,
                                                 float* grad_positions_device, void* cuda_stream);

/* The bounding-volume tree that mb2_character_closest_points_on_mesh_device searches, built from the current mesh faces over the host
 * array reference_positions [num_vertices][3] (normally the rest mesh) and replacing any earlier one; num_vertices == 0 with a null array
 * removes it. Only the topology is kept: each call refits the boxes to the instance's vertices, so the reference pose changes the speed of
 * the queries, never their results. No faces, num_vertices other than the faces', a null array or a non-finite position is
 * MB2_ERR_INVALID_ARGUMENT and leaves the earlier tree in place. Fresh device buffers and a device synchronisation before the old ones are
 * freed, as mb2_character_set_mesh_faces. mb2_character_set_mesh_faces drops the tree; mb2_character_clone copies it. */
int mb2_character_set_mesh_tree(mb2_character* c, int32_t num_vertices, const float* reference_positions);
/* The closest point on the mesh of each query point (pymomentum find_closest_points_on_mesh, array_kd_tree.cpp): for instance b and point
 * p = points[b][n], over the faces f of the mesh with vertices vertex_positions[b] ([B][V][3], V = the faces' num_vertices), the face with
 * the smallest (d2_f, f), d2_f = |q_f - p|^2 and (q_f, bary_f) the closest point of face f to p (Ericson 5.1.5, axel::projectOnTriangle),
 * among the candidates: faces with finite vertices and finite d2_f <= max_dist * max_dist (in float; max_dist may be +inf). Writes
 * out_points [B][N][3] = q, out_face [B][N] = f and out_bary [B][N][3]; without a candidate (a non-finite query included) -1 and zeros.
 * The result does not depend on the tree. Device memory on `cuda_stream`, asynchronous; batch == 0 or num_points == 0 is a no-op. No
 * faces or no tree, batch < 0, num_points < 0, a NaN or negative max_dist, a null pointer or a pointer that is not device memory on the
 * character's device is MB2_ERR_INVALID_ARGUMENT. Stream-ordered scratch from the device's default memory pool: the boxes of a slice of
 * instances, at most 256 MiB. No atomics: an instance gets the same bits alone as in any batch. */
int mb2_character_closest_points_on_mesh_device(const mb2_character* c, int32_t batch, int32_t num_points, const float* vertex_positions_device,
                                                const float* points_device, float max_dist, float* out_points_device, int32_t* out_face_device,
                                                float* out_bary_device, void* cuda_stream);

/* The closest target point of each query point (pymomentum find_closest_points, tensor_kd_tree.cpp / axel::SimdKdTree): for instance b
 * and query p = source[b][n], over the targets t_j = target[b or 0][j] (j = 0 .. M-1), the j with the smallest (d2_j, j),
 * d2_j = fmaf(dx, dx, fmaf(dy, dy, dz * dz)) with d = t_j - p, among the candidates: finite t_j with a finite d2_j <= max_dist * max_dist
 * (in float; max_dist may be +inf) and, when normals are given, dot(n_p, n_j) >= max_normal_dot (an fmaf chain; NaN fails). Writes
 * out_index [B][N] = j, out_points [B][N][3] = t_j and, with normals, out_normals [B][N][3] = n_j, copied bit for bit; without a
 * candidate (a non-finite query included) -1 and zeros. Points and normals are [B][N][3] / [B or 1][M][3] float32 device memory on
 * `device`; target_batched == 0 shares one target over the batch. The two normal arrays are both null (the plain variant) or both set
 * (with num_target == 0 the target arrays are not read and may be null), and out_normals is set exactly when normals are given. The result is a linear scan's, whatever the tree: each call builds, per target instance
 * and on `cuda_stream` with no host round trip, a tree over the target sorted by Morton code, in stream-ordered scratch of at most
 * 256 MiB per slice of instances. Asynchronous; batch == 0 or num_source == 0 is a no-op, num_target == 0 gives every query -1. A
 * negative device or size, a NaN or negative max_dist, a NaN max_normal_dot, a null or mismatched pointer or memory that is not device
 * memory on `device` is MB2_ERR_INVALID_ARGUMENT. No atomics: an instance gets the same bits alone as in any batch. */
int mb2_closest_points_device(int device, int32_t batch, int32_t num_source, int32_t num_target, int32_t target_batched,
                              const float* source_device, const float* source_normals_device, const float* target_device,
                              const float* target_normals_device, float max_dist, float max_normal_dot, float* out_points_device,
                              float* out_normals_device, int32_t* out_index_device, void* cuda_stream);

/* Input contraction of the implicit-function backward of solve_ik (diff_ik d_gradient_d_input_dot): for block `index` and every
 * instance b, the derivatives of grad_theta E_index(theta_b) . v_b with respect to the block's inputs, at the targets, constraint weights
 * and offsets the handle currently holds:
 *   grad_weights [B][nc]        w.r.t. the (per-instance) constraint weights
 *   grad_offsets [B][nc][3|4]   w.r.t. the offsets (orientation: the normalised quaternions the handle stores)
 *   grad_targets [B][nc][3|4]   w.r.t. the targets (idem)
 * for a Position block (shared or instanced) or an Orientation block (matrix difference, shared or instanced) with the L2 loss.
 * Entries of v for disabled parameters are ignored. Device memory in and out, asynchronous on `cuda_stream` (NULL = the legacy default
 * stream); a null output is skipped. Any other block kind or loss, an index out of range, a null parameters / direction pointer
 * (batch > 0) or memory that is not device memory on the function's device is MB2_ERR_INVALID_ARGUMENT. */
int mb2_solver_function_input_gradients_device(mb2_solver_function* f, int32_t index, const float* parameters_device /*[B][n]*/,
                                               const float* direction_device /*[B][n]*/, float* grad_weights_device, float* grad_offsets_device,
                                               float* grad_targets_device, void* cuda_stream);

/* Direction of the implicit-function backward of solve_ik: the reference's hessianInverseTimes
 * (diff_ik/fully_differentiable_body_ik.cpp:74-109) with the quantities d_modelParams_d_inputs (:112-238) needs beside it. For every
 * instance b, with E the enabled parameters, J_E the rows x |E| slice of the Jacobian at theta_b (the matrix
 * mb2_solver_function_get_jacobian_device writes; rows = the unpadded residual rows), r the residual and g = grad_parameters[b]
 * restricted to E:
 *   direction [B][n]                v_E = (2 J_E^T J_E)^+ g = 1/2 V diag(1 / s^2 if s^2 >= 1e-5, else 0) V^T g  (J_E = U S V^T, s^2
 *                                   compared in double); 0 on disabled parameters, and everywhere when E is empty
 *   jacobian_direction [B][rows8]   J v
 *   residual [B][rows8]             r
 *   gradient_rms [B]                sqrt(mean over E of (2 J_E^T r)^2), the RMS d_modelParams_d_inputs reports (0 when E is empty)
 * rows8 = mb2_solver_function_jacobian_rows (rows padded to 8; the padding rows are written 0). v then feeds
 * mb2_solver_function_input_gradients_device, and the per-block weight and target contractions follow from r and J v. The Jacobian
 * sweep and the solve (float64 Gram matrix on the smaller side of J_E, cyclic Jacobi eigen-solve) run on the device; device memory in
 * and out, asynchronous on `cuda_stream` (NULL = the legacy default stream), no host synchronisation. A null jacobian_direction,
 * residual or gradient_rms is skipped. A null parameters, gradient or direction pointer, or memory that is not device memory on the
 * function's device, is MB2_ERR_INVALID_ARGUMENT. The call uses the handle's Jacobian buffer: calls on the same handle must not overlap. */
int mb2_solver_function_implicit_direction_device(mb2_solver_function* f, const float* parameters_device /*[B][n]*/,
                                                  const float* grad_parameters_device /*[B][n]*/, float* direction_device /*[B][n]*/,
                                                  float* jacobian_direction_device /*[B][rows8]*/, float* residual_device /*[B][rows8]*/,
                                                  float* gradient_rms_device /*[B]*/, void* cuda_stream);

/* ---- GaussNewtonSolverT<float> x B (solver/gauss_newton_solver.h:67-137, solver/solver.h:36-100) ---- */
int mb2_solver_create(mb2_solver_function* f, const mb2_gauss_newton_options* opt, mb2_solver** out);
void mb2_solver_destroy(mb2_solver* s);
int mb2_solver_set_options(mb2_solver* s, const mb2_gauss_newton_options* opt); /* setOptions */
/* SolverT::setEnabledParameters — solver.cpp:41-48 (forwards to the solver function) */
int mb2_solver_set_enabled_parameters(mb2_solver* s, const uint64_t bits[MB2_PARAMETER_SET_WORDS]);
/* SolverT::solve for every instance — solver.cpp:50-128. parameters [B*n] in/out (host). errors[b] is
 * the objective before the last update (what solve() returns); iterations[b] = number of
 * doIteration calls; status[b] = mb2_instance_status. Any of errors/iterations/status may be NULL. */
int mb2_solver_solve(mb2_solver* s, float* parameters, double* errors, int32_t* iterations, int32_t* status);
/* The same call in two halves, for callers that keep several handles busy (e.g. the buckets of a mixed-rig batch): solve_async queues
 * the H2D copy, the solve and the D2H copy on the handle's stream and returns (use pinned host memory for a truly asynchronous copy);
 * wait blocks until they are done and returns the per-instance results. */
int mb2_solver_solve_async(mb2_solver* s, float* parameters);
int mb2_solver_wait(mb2_solver* s, double* errors, int32_t* iterations, int32_t* status);
/* Same with parameters resident on the device, on `cuda_stream` (NULL = handle stream). Results are fetched with
 * mb2_solver_get_results after synchronising. The fused single-kernel path (default options on a rig whose tiles fit in shared
 * memory, no line search) is fully asynchronous; the multi-kernel path is asynchronous up to min_iterations and then reads the
 * device-side active counter every fourth iteration (a host round trip on `cuda_stream`) so that a converged batch stops early. */
int mb2_solver_solve_device(mb2_solver* s, float* parameters_device, void* cuda_stream);
int mb2_solver_get_results(mb2_solver* s, double* errors, int32_t* iterations, int32_t* status);
/* getErrorHistory (solver.h:90): [B][max_iterations], valid up to iterations[b] */
int mb2_solver_get_error_history(mb2_solver* s, double* history);
/* sum over the batch of iterations executed / kernels launched by the last solve (for throughput) */
int mb2_solver_get_counters(mb2_solver* s, uint64_t* total_iterations, uint64_t* kernel_launches);
/* device time of the dominant kernels in the last solve, milliseconds (CUDA events on the handle's
 * stream); index: 0 = FK+Jacobian, 1 = JtJ/Jtr, 2 = Cholesky/update, 3 = error-only. Enabled by
 * mb2_solver_set_profiling(s, 1); off by default (events serialise the stream). Level 2 additionally runs the instrumented
 * instantiations of the fused kernels (per-phase SM cycles, mb2_solver_get_fused_profile); those are slower, so take kernel times
 * at level 1 and phase shares at level 2. */
int mb2_solver_set_profiling(mb2_solver* s, int32_t enabled);
int mb2_solver_get_phase_times(mb2_solver* s, double ms[4], uint64_t launches[4]);
/* Per-instance algorithmic sizes of the plan the last solve ran on (roofline accounting in bench.py; no reference
 * counterpart): [0] structurally non-zero Jacobian entries written per iteration, [1] device Jacobian columns (without
 * the residual column), [2] ldJ, [3] parameters in the normal equations (ns), [4] 16x16 tiles held by the tile-sparse
 * Cholesky (0: dense Eigen-structured kernel), [5] tile multiply-accumulate blocks per factorisation, [6] levels of the
 * tile elimination tree, [7] residual rows m (row groups aligned to 4 in the strip layout), [8] floats per instance of the Jacobian in
 * strip layout (0: K-major matrix), [9] multiply-accumulates per instance of the tile-sparse Gram kernel, [10] its strip pairs,
 * [11] instance groups per CTA of the fused persistent kernel (0: the plan does not fit / was not built for it). */
int mb2_solver_get_plan_stats(mb2_solver* s, int64_t stats[12]);
/* Which fused kernel the last solve ran (fused: 0 none, 1 persistent whole-solve kernel, 2 Gram + Cholesky per iteration) and, after
 * mb2_solver_set_profiling(s, 1), its device time and the per-phase SM cycles of one instance group (persistent kernel: over its whole
 * share of the batch; Gram + Cholesky: CTA 0 summed over the iterations, [0] = prologue, [1..4] unused): [0] work fetch + theta load, [1] ParameterTransform
 * + strip zero fill, [2] FK sweep, [3] residual/units, [4] Jacobian cells, [5] Gram (J^T J, J^T r), [6] parked tiles written over the strips,
 * [7] Cholesky diagonal tiles, [8] panel tiles, [9] updates, [10] backward substitution, [11] update + bookkeeping + write-back.
 * groups = instance groups per CTA of the persistent kernel. Any output pointer may be NULL. No reference counterpart. */
int mb2_solver_get_fused_profile(mb2_solver* s, int32_t* fused, int32_t* groups, double* kernel_ms, uint64_t phase_cycles[12]);
/* Which variant of the FK + residual sweep the handle last launched, for the Jacobian sweep (jacobian != 0: get_jacobian[_device],
 * get_jtjr, the implicit direction, a solver's per-iteration Jacobian pass) or the error-only sweep (jacobian == 0: get_error,
 * get_skeleton_state, a solver's line-search trials): [0] table staging (1 every read-only table in shared memory, 2 all but the
 * Jacobian cells and chain-rule contributions, 0 none), [1] warps per instance (1, 2, 4 or 8), [2] instances per CTA, [3] CTAs,
 * [4] dynamic shared memory per CTA in bytes. All zero before the first such sweep and after a sweep whose instance does not fit in
 * shared memory (the entry that launched it failed). The fused persistent kernel runs its own sweep and records nothing here.
 * No reference counterpart. */
int mb2_solver_function_get_sweep_launch(mb2_solver_function* f, int32_t jacobian, int64_t out[5]);
/* What the character operations' per-instance kernels would launch for `batch` instances, planned by the code that launches them and
 * with nothing enqueued. op: 0 model_parameters_to_skeleton_state, 1 joint_parameters_to_skeleton_state, 2 model_parameters_to_positions,
 * 3 joint_parameters_to_positions (num_points points); backward != 0: their backward. out: [0] warps per instance W (1, 2, 4 or 8),
 * [1] instances per CTA, [2] threads per CTA, [3] CTAs, [4] dynamic shared memory per CTA in bytes, [5] 1 when the point tables are
 * staged in shared memory. All zero when nothing runs (batch 0, positions with no point). An instance that does not fit in shared
 * memory next to the tables is refused with MB2_ERR_CUDA, as the operation refuses it. The shared-offset positions backward launches
 * per slice of the batch when its per-instance offset rows exceed 256 MiB of scratch: this reports one launch of `batch` instances.
 * No reference counterpart. */
int mb2_character_get_instance_launch(const mb2_character* c, int32_t op, int32_t backward, int32_t batch, int32_t num_points, int64_t out[6]);
/* The same record for mb2_solver_function_input_gradients_device over the function's batch ([5] is 0). No reference counterpart. */
int mb2_solver_function_get_input_gradient_launch(mb2_solver_function* f, int64_t out[6]);
/* The linear-solve path the solver's last solve ran, as one host function chose it (the CPU emulator of the tests runs the same
 * choice): [0] kind (1 JtJ + dense Eigen-structured Cholesky, 2 JtJ + tile-scheduled Cholesky, 3 tile-sparse Gram + tile Cholesky
 * in two launches, 4 Gram + Cholesky in one launch, 5 the persistent kernel, 6 QR, 7 trust-region QR), [1] plan mode (1 compact
 * columns, 2 tile schedule), [2] dense tile pattern, [3] Jacobian in strips, [4] mb2_jtj_mode after AUTO, [5] dense Cholesky block
 * size NB, [6] its matrix in shared memory, [7] / [8] threads of the Gram / tile Cholesky kernels (256 or 512), [9] Jacobian rows
 * the QR kernels fold at once (the limit), [10] QR row chunks, [11] rows of the widest chunk, [12] floats of the trust-region R kept
 * per instance, [13] instance groups per CTA of the persistent kernel (any plan with strips), [14] its dynamic shared memory in
 * bytes. All zero before the first solve and after a refused solve (by its options, or no resident Gram + Cholesky CTA); a CUDA error
 * later in a solve leaves the path it had chosen. No reference counterpart. */
int mb2_solver_get_solve_path(mb2_solver* s, int64_t out[15]);

/* ---- Mixed-rig batches (BASELINE.json configs[4]): heterogeneous instances -> buckets sharing one plan -> batched solves --------
 * The reference treats a batch element by element (pymomentum/tensor_ik/tensor_ik.cpp:127-177 builds error functions, solver function
 * and solver per element). Here instances are bucketed by (rig, constraint parents): inside a bucket offsets, targets, weights and
 * the number of constraints are per instance (shorter instances are padded with zero-weight constraints, at most granule - 1 of them),
 * every bucket is one batched solve, results come back in input order. Position constraints (+ optionally the rig's ParameterLimits). */
typedef struct mb2_mixed_batch mb2_mixed_batch;
const char* mb2_mixed_batch_last_error(void);
int mb2_mixed_batch_create(int device, int32_t granule /*constraints; <= 0: 8*/, mb2_mixed_batch** out);
void mb2_mixed_batch_destroy(mb2_mixed_batch* b);
/* the character must outlive the batch (ownership as everywhere in momentum: non-owning references) */
int mb2_mixed_batch_add_rig(mb2_mixed_batch* b, const mb2_character* c, int32_t num_parameters, int32_t* rig_id);
int mb2_mixed_batch_use_limits(mb2_mixed_batch* b, int32_t enabled, float weight); /* LimitErrorFunctionT over each rig's limits */
int mb2_mixed_batch_add_instance(mb2_mixed_batch* b, int32_t rig_id, int32_t num_constraints, const int32_t* parents, const float* offsets /*[nc*3]*/,
                                 const float* weights /*[nc]*/, const float* targets /*[nc*3]*/, const float* theta0 /*[n of the rig]*/, int32_t* instance_id);
int mb2_mixed_batch_set_parameters(mb2_mixed_batch* b, int32_t instance_id, const float* theta0);
int mb2_mixed_batch_solve(mb2_mixed_batch* b, const mb2_gauss_newton_options* opt);
int mb2_mixed_batch_get_result(mb2_mixed_batch* b, int32_t instance_id, float* theta, double* error, int32_t* iterations, int32_t* status);
int mb2_mixed_batch_get_results(mb2_mixed_batch* b, float* theta, const int64_t* theta_offsets, double* errors, int32_t* iterations, int32_t* status);
/* [0] instances, [1] buckets, [2] residual rows before padding, [3] after, [4] largest bucket, [5] singleton buckets */
int mb2_mixed_batch_stats(mb2_mixed_batch* b, int64_t stats[6]);
/* [0] rig, [1] instances, [2] constraints (padded), [3] Gauss-Newton iterations of the last solve */
int mb2_mixed_batch_bucket_info(mb2_mixed_batch* b, int32_t bucket, int64_t info[4]);

/* ---- single-process multi-GPU: one batch sharded over several devices (SURVEY 8e; north_star "host code stays C++") ----
 * The reference solves a batch element by element on host threads (pymomentum/tensor_ik/tensor_ik.cpp:127-177, dispenso::parallel_for);
 * instances are independent, so a batch of total_batch instances is cut into contiguous blocks, one per device, each block an ordinary
 * mb2_solver on its own device driven by its own host thread. There is no data-path collective: the only cross-device quantity is the
 * aggregate {sum of final errors, total iterations, instances that ended with status OK}, summed on the host from the per-instance
 * results (the 24-byte all-reduce of SURVEY 8e; with one process there is nothing to send over NVLink).
 *
 * Replicas: mb2_character_clone puts the rig on another device; mb2_solver_function_clone copies the DEFINITION of a solver function
 * (error-function blocks, shared constraint weights, block weights, enabled parameters - no targets) for a new batch size. */
int mb2_character_clone(const mb2_character* c, int device, mb2_character** out);
int mb2_solver_function_clone(const mb2_solver_function* f, const mb2_character* c_on_device, int32_t batch, mb2_solver_function** out);
int mb2_character_device(const mb2_character* c);
const mb2_character* mb2_solver_function_character(const mb2_solver_function* f);
int32_t mb2_solver_function_num_error_functions(const mb2_solver_function* f);
int32_t mb2_solver_function_target_size(const mb2_solver_function* f, int32_t index); /* floats per instance of block `index` */

typedef struct mb2_sharded_solver mb2_sharded_solver;
const char* mb2_sharded_last_error(void);
/* `prototype` defines the problem (it is only read, on its own device, and may be destroyed afterwards); devices[] may name a device more
 * than once (several shards on one GPU). Shard k holds instances [first_k, first_k + count_k), count = total_batch / num_devices rounded
 * so that the counts differ by at most one. */
int mb2_sharded_solver_create(const mb2_solver_function* prototype, int32_t total_batch, int32_t num_devices, const int32_t* devices,
                              const mb2_gauss_newton_options* opt, mb2_sharded_solver** out);
void mb2_sharded_solver_destroy(mb2_sharded_solver* s);
int32_t mb2_sharded_solver_num_shards(const mb2_sharded_solver* s);
int mb2_sharded_solver_shard_info(const mb2_sharded_solver* s, int32_t shard, int32_t info[3] /* device, first instance, count */);
int mb2_sharded_solver_set_options(mb2_sharded_solver* s, const mb2_gauss_newton_options* opt);
/* targets[total_batch][size of block index] in instance order, host memory (SkeletonErrorFunction::setConstraints per instance) */
int mb2_sharded_solver_set_targets(mb2_sharded_solver* s, int32_t index, const float* targets);
/* SolverT::solve over the whole batch: parameters[total_batch * n] in/out (host), per-instance results optional */
int mb2_sharded_solver_solve(mb2_sharded_solver* s, float* parameters, double* errors, int32_t* iterations, int32_t* status);
/* aggregate of the last solve: [0] sum of final errors, [1] total Gauss-Newton iterations, [2] instances with status MB2_INSTANCE_OK */
int mb2_sharded_solver_get_aggregate(const mb2_sharded_solver* s, double aggregate[3]);

#ifdef __cplusplus
}
#endif
#endif /* MOMENTUM_B200_H_ */
