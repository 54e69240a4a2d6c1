/*
 * fn2_solver.h -- C-ABI of libfn2.so's solver: Caffe's SGD and Adam solvers over a TRAIN net created through fn2.h
 * (reference: include/caffe/solver.hpp, include/caffe/sgd_solvers.hpp, src/caffe/solver.cpp:194-481,
 * src/caffe/solvers/sgd_solver.cpp, adam_solver.cpp).  fn2.h and this header together state the ABI; the conventions are
 * fn2.h's: status 0 or negative with the message in fn2_last_error(), and the size query for outputs (out == NULL reports
 * *bytes, a text output counts its NUL).
 *
 * Solver text is a solver prototxt (caffe.proto:104-244).  Supported: type SGD and Adam (the deprecated solver_type enum is
 * upgraded like upgrade_proto.cpp:1002-1037), the seven lr_policy values of SGDSolver::GetLearningRate, base_lr, gamma,
 * power, stepsize, stepvalue, max_iter, momentum, momentum2, delta, weight_decay, regularization_type (L2, L1),
 * clip_gradients, iter_size, average_loss, snapshot, snapshot_prefix, snapshot_after_train.  Accepted with no effect: net,
 * train_net, display, debug_info, solver_mode GPU, device_id, random_seed.  Refused with a message naming the field: other
 * solver types, test nets, snapshot_format HDF5, snapshot_diff, solver_mode CPU, an unknown lr_policy or regularization_type.
 */
#ifndef FN2_SOLVER_H_
#define FN2_SOLVER_H_

#include "fn2.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fn2_solver fn2_solver;

/* A solver over `net` (created with phase TRAIN; it must outlive the solver).  Allocates the history and the segment table
 * of the trainable parameters (lr_mult != 0) once. */
FN2_API int fn2_solver_create(const char* solver_text, fn2_net* net, fn2_solver** out);
FN2_API void fn2_solver_destroy(fn2_solver* solver);
/* SGDSolver::ApplyUpdate (sgd_solver.cpp:102-116) for the current iteration, enqueued on the net's stream as one fused pass
 * over the parameter arena (plus two small kernels when clip_gradients >= 0), then iter += 1.  The parameter diffs are
 * expected to hold the gradients summed over iter_size forward/backward passes; they are left holding the applied update.
 * Parameters with lr_mult == 0 are not touched and their history stays zero. */
FN2_API int fn2_solver_apply_update(fn2_solver* solver);
/* Number of updates applied (Solver::iter) and the multistep position (current_step). */
FN2_API int fn2_solver_iter(fn2_solver* solver, int* iter, int* current_step);
/* Loss weights of the net's outputs in output order (Net::blob_loss_weights), for the loss the solver reports. */
FN2_API int fn2_solver_output_loss_weights(fn2_solver* solver, float* weights, int n);
/* The SolverState message (caffe.proto:247-252) as bytes: iter, learned_net (the .caffemodel file name to record),
 * history in Net::learnable_params order (Adam: every m, then every v), current_step.  Size query. */
FN2_API int fn2_solver_state(fn2_solver* solver, const char* learned_net, void* out, size_t* bytes);
/* RestoreSolverStateFromBinaryProto (sgd_solver.cpp:305-322) from SolverState bytes: iter, current_step and the history.
 * The weights named by learned_net are the caller's to load (fn2_solverstate_learned_net, fn2_net_copy_trained_layers). */
FN2_API int fn2_solver_restore(fn2_solver* solver, const void* state, size_t bytes);
/* learned_net of SolverState bytes, as text.  Size query. */
FN2_API int fn2_solverstate_learned_net(const void* state, size_t n, char* out, size_t* bytes);
/* SGDSolver::GetLearningRate (sgd_solver.cpp:27-63) at `iter`, on the host: *current_step is read and, for multistep,
 * advanced by at most one step, as the solver does once per iteration.  Validates the whole solver text. */
FN2_API int fn2_solver_learning_rate(const char* solver_text, int iter, int* current_step, float* rate);
/* The resolved parameters of solver text (type upgraded, defaults filled) as `name: value` lines.  Size query. */
FN2_API int fn2_solver_params(const char* solver_text, char* out, size_t* bytes);

#ifdef __cplusplus
}
#endif

#endif /* FN2_SOLVER_H_ */
