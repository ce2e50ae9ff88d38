// Host-side model of a character and of the batched solver function's objective, and the planner
// that flattens it into the unit / cell / contribution tables consumed by the device sweep.
//
// The planner performs, once per (constraint topology, enabled-parameter set), the ancestor walks
// that the reference repeats for every constraint on every iteration
// (joint_error_function-inl.h:229-294, state_error_function.cpp:486-555, limit_error_function.cpp:740-777),
// including its gating rules (activeJointParams_, enabledParameters_, zero weights).
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "ik_chol_sched.h"
#include "ik_types.h"

namespace mb2 {

struct HostLimit { // character/parameter_limits.h:117-127, flattened like mb2_parameter_limit
  int32_t type;
  float weight;
  int32_t i[4];
  float f[27];
};

struct HostCharacter {
  int32_t numJoints{0}, numParams{0};
  std::vector<int32_t> parent;
  std::vector<float> offset, prerot;
  std::vector<int32_t> ptOuter, ptInner;
  std::vector<float> ptVals, ptOffsets;
  std::vector<HostLimit> limits;
  // derived
  std::vector<int32_t> levelStart, levelJoints;
  // the reverse sweep of the skeleton-state backward: children of each joint (CSR, ascending), and the ParameterTransform by model
  // parameter (CSC, rows ascending within a column)
  std::vector<int32_t> childStart, children;
  std::vector<int32_t> ptColStart, ptColRows;
  std::vector<float> ptColVals;
  std::string validate() const; // empty when fine (MT_CHECK-style message otherwise)
  void buildLevels();
  void buildBackwardTables();
  // ParameterTransformT::computeActiveJointParams (parameter_transform.cpp:97-107)
  std::vector<uint8_t> computeActiveJointParams(const std::vector<uint8_t>& enabled) const;
};

// Linear-blend skinning of a character (SkinWeights + Character::inverseBindPose, skin_weights.h:19-40, character.h), flattened into
// the tables of SkinTables (ik_types.h). Built and validated by makeSkinning only.
struct HostSkinning {
  int32_t numVertices{0};
  std::vector<float> restVertices;             // [V][3]
  std::vector<int32_t> vertStart, vertJoint;   // by vertex, active slots only
  std::vector<float> vertWeight;
  std::vector<float> inverseBindPose;          // [J][12]
  std::vector<int32_t> jointStart, infVertex;  // by joint, vertices ascending
  std::vector<float> infWeight;
  std::vector<int32_t> segStart, segJoint, jointSegStart;
  int32_t numInfluences() const { return int32_t(vertJoint.size()); }
  int32_t numSegments() const { return int32_t(segJoint.size()); }
};

struct HostErrorFunction {
  int32_t kind{0}; // 0 position, 1 orientation, 2 orientation rot-diff, 3 state, 4 limit, 5 plane, 6 model parameters
  float weight{1.f};
  float lossAlpha{2.f}, lossC{1.f};
  std::vector<int32_t> parents;
  std::vector<float> offsets; // 3 or 4 per constraint
  std::vector<float> weights; // shared constraint weights
  int32_t rotationErrorType{0};
  float posWgt{1.f}, rotWgt{1.f};
  std::vector<float> posW, rotW;
  bool halfPlane{false};            // plane: PlaneErrorFunctionT(above)
  bool instanceOffsets{false};      // position / orientation: offsets are per instance (record per constraint = target, then offset)
  std::vector<float> paramWeights; // model parameters: targetWeights_ [numParams]
  // layout (assigned when added)
  int32_t targetOff{0}, targetSize{0}; // floats per instance
  int32_t weightOff{0};                // into the constraint-weight array
  int32_t numConstraints() const { return int32_t(parents.size()); }
};

// The host description of a solver function: its blocks, the per-instance layout of their targets and constraint weights, and the
// enabled parameters.
struct HostFunction {
  std::vector<HostErrorFunction> efs;
  std::vector<uint8_t> enabled;     // [numParams]
  int32_t targetStride{0};          // target floats per instance
  int32_t numWeights{0};            // constraint weights per instance
  std::vector<float> weights;       // the shared constraint weights [numWeights]
  bool weightsPerInstance{false};
  // Appends a block and assigns its target and weight offsets; *index = its position. A block with constraint weights cannot follow
  // per-instance weights (their [B][numWeights] layout is fixed).
  std::string add(const HostErrorFunction& ef, int32_t* index);
  int32_t actualParameters() const;                       // last enabled parameter + 1 (skeleton_solver_function.cpp:45-52)
  int32_t jacobianRows(const HostCharacter& ch) const;    // getJacobianBlockSize of the blocks with weight > 0, padded to 8 (solver_function.cpp:33-38)
  int32_t jacobianStride(const HostCharacter& ch) const;  // leading dimension of a K-major device Jacobian column
};

// ---- Characters and error-function blocks from the C-ABI arrays (mb2_character_*, mb2_add_*_error_function) ----
// Each returns an empty string when the arguments are accepted, else the message of the first rejected one.
std::string makeCharacter(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams, const int32_t* outer,
                          const int32_t* inner, const float* vals, const float* ptOffsets, HostCharacter& out); // validated, tree levels built
// CharacterTables on the host copy (the CPU emulators' view of what mb2_character::tables gives the kernels)
CharacterTables hostCharacterTables(const HostCharacter& ch);
std::string setParameterLimits(HostCharacter& ch, int32_t count, const mb2_parameter_limit* limits);
// restVertices [V][3], skinIndex / skinWeight [V][8], inverseBindPose [J][12]. A vertex's influences end at its first zero weight
// (linear_skinning.cpp:76-80); the slots after it are ignored whatever they hold.
std::string makeSkinning(const HostCharacter& ch, int32_t numVertices, const float* restVertices, const int32_t* skinIndex, const float* skinWeight,
                         const float* inverseBindPose, HostSkinning& out);
std::string positionErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t nc, const int32_t* parents, const float* offsets,
                                  const float* weights, HostErrorFunction& out);
std::string instancedPositionErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t nc, const int32_t* parents, const float* weights,
                                           HostErrorFunction& out);
std::string planeErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t above, int32_t nc, const int32_t* parents, const float* offsets,
                               const float* weights, HostErrorFunction& out);
std::string modelParametersErrorFunction(const HostCharacter& ch, float weight, const float* targetWeights, HostErrorFunction& out);
std::string orientationErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t rotDiff, int32_t nc, const int32_t* parents,
                                     const float* offsets, const float* weights, HostErrorFunction& out);
// record per constraint = target xyzw, offset xyzw (both normalised when uploaded)
std::string instancedOrientationErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t rotDiff, int32_t nc, const int32_t* parents,
                                              const float* weights, HostErrorFunction& out);
std::string stateErrorFunction(const HostCharacter& ch, float weight, int32_t rotationErrorType, float posWgt, float rotWgt, const float* posW, const float* rotW,
                               HostErrorFunction& out);
std::string limitErrorFunction(float weight, float alpha, float c, HostErrorFunction& out);

struct Plan {
  std::vector<EfDesc> efs;
  std::vector<UnitDesc> units;
  std::vector<CellDesc> cells;
  std::vector<ContribDesc> contribs;
  std::vector<float> limitData;
  int32_t numRows{0};   // m, unpadded (sum of getJacobianBlockSize of blocks with weight > 0)
  int32_t recStride{0};
  int32_t actualParameters{0}; // skeleton_solver_function.cpp:45-52
  std::vector<int32_t> enabledList; // gauss_newton_solver.cpp:57-66
  int32_t numCols{0};   // device Jacobian columns: numParams (full) or enabledList.size() (compact)
  bool compact{false};
  std::vector<int32_t> deviceCols; // [numCols] model parameter held by each device column
};

// Builds the plan. `enabled` has numParams entries.
// compact = true drops the columns of disabled parameters and packs the enabled ones in order (what the solver
// needs: gauss_newton_solver.cpp:204-209 discards the others anyway); compact = false keeps the reference's
// full column positions (getJacobian / getJtJR parity).
// alignRowGroups: every multi-row unit starts on a row that is a multiple of 4 (the rows in between stay zero), so that four
// consecutive rows of a column are one aligned 16-byte piece of the K-major device Jacobian (tile-sparse Gram kernel).
// columnOrder (optional, compact only): model parameters in the order the device columns should take (a permutation
// of the enabled parameters, e.g. the Cholesky elimination order); default = ascending enabled parameters.
std::string buildPlan(const HostCharacter& ch, const std::vector<HostErrorFunction>& efs, const std::vector<uint8_t>& enabled, bool compact, Plan& out,
                      const std::vector<int32_t>* columnOrder = nullptr, bool alignRowGroups = false);

// getJacobianSize() of a block (joint_error_function-inl.h:300-302, state_error_function.cpp:394-404,
// limit_error_function.cpp:1138-1161)
int32_t jacobianBlockSize(const HostCharacter& ch, const HostErrorFunction& ef);

// MB2_CHOLESKY_AUTO: the tile schedule on the sparse pattern from 48 enabled parameters up, the dense Eigen-structured kernel below.
int resolveCholeskyMode(int requested, const std::vector<uint8_t>& enabled);

// Planning of the tile-scheduled solver path, which fixes the data layout every tile kernel reads:
//   1. the compact plan in natural column order; 2. the elimination order (ties broken by joint depth) and the tile schedule over it
//   (densePattern: every tile present); 3. the device columns in elimination order (layoutDeviceColumns); 4. the plan re-built on those
//   columns, with multi-row units on row quads when `strips`; 5. with strips, the Gram plan, and each cell's strip offset and quad stride
//   patched into the plan. `gram` stays empty without strips.
std::string planSolverPath(const HostCharacter& ch, const std::vector<HostErrorFunction>& efs, const std::vector<uint8_t>& enabled, bool densePattern, bool strips,
                           Plan& plan, CholSchedule& sched, GramPlan& gram);

} // namespace mb2
