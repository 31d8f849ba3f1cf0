// TEST INFRASTRUCTURE ONLY — host build of the step loop of the L-BFGS form of the cluster kernel
// (pydens_b200/csrc/pinn_small_lbfgs.cuh) over the state machine of pinn_lbfgs.cuh in fp64, so that the loop can be
// checked against torch.optim.LBFGS on a machine without a GPU.  Never loaded by the product.
#include <stddef.h>
#include "../../pydens_b200/csrc/pinn_lbfgs.cuh"

using namespace pinn::lbfgs;

extern "C" size_t lbfgs_steps_state_bytes(int64_t n, int history_size) { return state_bytes<double>(n, history_size); }

// Step s of a launch keeps the batch of step number step0 + s (step0: the counter when the launch begins) for all of
// its evaluations, and evaluation and advance alternate until the state machine ends the step, which logs its first
// loss and advances the counter.  `objective(step, params, grads_and_loss, ctx)` evaluates [grads | loss] on that
// step's batch.  -> the evaluations made
typedef void (*lbfgs_steps_objective)(uint64_t step, const double* params, double* grads_and_loss, void* ctx);
extern "C" int lbfgs_steps_run(const PinnLbfgs* c, int64_t n, double* params, void* state, const double* mask,
                               int n_steps, lbfgs_steps_objective objective, void* ctx, double* grads_and_loss) {
    const uint64_t step0 = *c->step_counter;
    int evals = 0;
    for (int s = 0; s < n_steps; ++s) {
        for (;;) {
            objective(step0 + (uint64_t)s, params, grads_and_loss, ctx);
            ++evals;
            if (advance_host(*c, n, params, grads_and_loss, state, mask) == PINN_LBFGS_DONE) break;
        }
    }
    return evals;
}

// the layout of PinnLbfgsMember as gcc sees it: size, then the offset of every field in declaration order
#define MOFF(f) (int64_t) offsetof(PinnLbfgsMember, f)
extern "C" int lbfgs_steps_member_layout(int64_t* out) {
    int64_t v[] = {(int64_t)sizeof(PinnLbfgsMember), MOFF(params), MOFF(state), MOFF(mask), MOFF(points), MOFF(seed),
                   MOFF(step_counter), MOFF(losses_ring), MOFF(lr)};
    int k = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < k; ++i) out[i] = v[i];
    return k;
}
