// Solver: Caffe's SGD and Adam solvers (reference: include/caffe/solver.hpp, include/caffe/sgd_solvers.hpp,
// src/caffe/solver.cpp, src/caffe/solvers/sgd_solver.cpp, adam_solver.cpp) over an existing TRAIN Net.  What runs here is
// ApplyUpdate and the solver state; the Step / Solve / Snapshot loop around it (forward, backward, callbacks, files) is the
// Python front end's, like pycaffe's.
#pragma once
#include "net.hpp"
#include "solver_update.hpp"

namespace caffe {

class Solver {
 public:
    // Validates the parameters (Validate) and builds the segment table and history once; a warm ApplyUpdate allocates nothing.
    Solver(const SolverParameter& param, Net<float>* net);

    // Refuses, naming the field, what this solver does not do: other solver types, test nets, HDF5 snapshots, snapshot_diff,
    // solver_mode CPU, an unknown lr_policy or regularization_type.
    static void Validate(const SolverParameter& param);
    // SGDSolver::GetLearningRate (sgd_solver.cpp:27-63) at `iter`; multistep advances *current_step by at most one step.
    static float LearningRate(const SolverParameter& param, int iter, int* current_step);

    // ClipGradients, then Normalize / Regularize / ComputeUpdateValue of every trainable parameter and Net::Update, enqueued on
    // the net's stream; then iter += 1 (solver.cpp:241-246).
    void ApplyUpdate();
    int iter() const { return iter_; }
    int current_step() const { return current_step_; }

    // SnapshotSolverStateToBinaryProto / RestoreSolverStateFromBinaryProto (sgd_solver.cpp:260-322).  History order:
    // Net::learnable_params order; Adam: every m, then every v.
    std::string State(const std::string& learned_net);
    void Restore(const void* bytes, size_t n);

 private:
    SolverParameter param_;
    Net<float>* net_;
    bool adam_;
    int iter_ = 0, current_step_ = 0;
    vector<Net<float>::LearnableParam> params_;
    vector<int> trainable_;                    // learnable ids with lr_mult != 0
    vector<fn2::SolverSegment> segs_;          // one per trainable id
    int nchunks_ = 0;
    size_t hist_floats_ = 0;
    DeviceBuffer segs_dev_, chunks_dev_, hist0_, hist1_, partial_, scale_;
};

}  // namespace caffe
