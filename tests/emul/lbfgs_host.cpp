// TEST INFRASTRUCTURE ONLY — host build of the L-BFGS state machine (pydens_b200/csrc/pinn_lbfgs.cuh) in fp64, so that
// its control logic and vector passes can be checked against torch.optim.LBFGS on a machine without a GPU.  Never
// loaded by the product.
#include <stddef.h>
#include "../../pydens_b200/csrc/pinn_lbfgs.cuh"

using namespace pinn::lbfgs;

extern "C" size_t lbfgs_host_state_bytes(int64_t n, int history_size) { return state_bytes<double>(n, history_size); }
extern "C" size_t lbfgs_host_vector_offset(int history_size) { return vector_offset(history_size); }

extern "C" int lbfgs_host_advance(const PinnLbfgs* c, int64_t n, double* params, const double* grads_and_loss,
                                  void* state, const double* mask) {
    return advance_host(*c, n, params, grads_and_loss, state, mask);
}

// the layout of the state header as gcc sees it: size, then the offset of every field in declaration order
#define OFF(f) (int64_t) offsetof(PinnLbfgsState, f)
extern "C" int lbfgs_host_header_layout(int64_t* out) {
    int64_t v[] = {(int64_t)sizeof(PinnLbfgsState), OFF(n_iter), OFF(func_evals), OFF(t), OFF(H_diag), OFF(prev_loss),
                   OFF(ring_count), OFF(ring_head), OFF(phase), OFF(cur_iter), OFF(current_evals), OFF(opt_cond),
                   OFF(g_src), OFF(action), OFF(act_arg), OFF(act_eval), OFF(loss), OFF(first_loss), OFF(gtd),
                   OFF(d_norm), OFF(gsum_g), OFF(hg), OFF(ls_iter), OFF(ls_evals), OFF(max_ls), OFF(ls_done),
                   OFF(ls_zoom), OFF(insuf), OFF(low), OFF(high), OFF(gp_ref), OFF(new_ref), OFF(t_prev), OFF(f_prev),
                   OFF(gtd_prev), OFF(f_new), OFF(gtd_new), OFF(br_t), OFF(br_f), OFF(br_gtd), OFF(br_g), OFF(ref_gmax),
                   OFF(r_dot), OFF(r_max), OFF(r_l1)};
    int k = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < k; ++i) out[i] = v[i];
    return k;
}

#define COFF(f) (int64_t) offsetof(PinnLbfgs, f)
extern "C" int lbfgs_host_cfg_layout(int64_t* out) {
    int64_t v[] = {(int64_t)sizeof(PinnLbfgs), COFF(lr), COFF(tolerance_grad), COFF(tolerance_change), COFF(max_iter),
                   COFF(max_eval), COFF(history_size), COFF(line_search), COFF(mask), COFF(losses_ring), COFF(ring_len),
                   COFF(step_counter)};
    int k = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < k; ++i) out[i] = v[i];
    return k;
}
