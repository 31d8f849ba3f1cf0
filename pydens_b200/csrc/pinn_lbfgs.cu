// pinn_lbfgs_advance: one CTA runs the L-BFGS state machine of pinn_lbfgs.cuh between two evaluations of the objective.
// Thread 0 runs the control; all threads run the vector passes it asks for.  The state header is held in shared
// memory for the launch; the Gram entries and the vectors stay in the state buffer.  Where 3 n_params floats fit, the
// history pass stages g, y and s in shared memory, since every warp reads them once per history pair it reduces.
#include <cuda_runtime.h>
#include <stdio.h>
#include <atomic>
#include "pinn_lbfgs.cuh"

extern int pinn_fail_message(int code, const char* msg);

namespace pinn {
namespace lbfgs {

static const int THREADS = 512;
static const int STAGE_MAX_BYTES = 192 * 1024;

__global__ void __launch_bounds__(THREADS, 1)
lbfgs_advance_kernel(const PinnLbfgs c, int64_t n, float* params, const float* out, void* state, int* status,
                     int stage_on) {
    extern __shared__ __align__(16) float lb_stage[];
    __shared__ PinnLbfgsState h;
    __shared__ double red[THREADS / 32 + 1];
    View<float> v(state, n, c.history_size);
    CtaExec ex(red);
    if (threadIdx.x == 0) h = *(const PinnLbfgsState*)state;
    __syncthreads();
    const double loss = (double)out[n];
    for (;;) {
        if (threadIdx.x == 0) lbfgs_control(c, &h, v.sy, v.yy, loss, v.S);
        __syncthreads();
        const int a = h.action, eval = h.act_eval;
        if (a == ACT_DONE) break;
        lbfgs_pass(ex, c, &h, v, n, params, out, c.mask, stage_on ? lb_stage : (float*)nullptr);
        __syncthreads();
        if (a == ACT_MOVE && eval) break;
    }
    if (threadIdx.x == 0) {
        *(PinnLbfgsState*)state = h;
        *status = h.action == ACT_DONE ? PINN_LBFGS_DONE : PINN_LBFGS_EVALUATE;
    }
}

}  // namespace lbfgs
}  // namespace pinn

using namespace pinn::lbfgs;

extern "C" size_t pinn_lbfgs_state_bytes(int64_t n_params, int history_size) {
    if (n_params < 1 || history_size < 1) return 0;
    return state_bytes<float>(n_params, history_size);
}

extern "C" size_t pinn_lbfgs_vector_offset(int history_size) {
    return history_size < 1 ? 0 : vector_offset(history_size);
}

extern "C" int pinn_lbfgs_advance(const PinnLbfgs* cfg, int64_t n_params, float* params, const float* grads_and_loss,
                                  void* state, int* status, void* stream) {
    if (!cfg || !params || !grads_and_loss || !state || !status || !cfg->mask || !cfg->step_counter)
        return pinn_fail_message(PINN_E_INVALID, "pinn_lbfgs_advance: null argument");
    if (n_params < 1 || !(cfg->lr >= 0) || cfg->max_iter < 1 || cfg->max_eval < 1 || cfg->history_size < 1
            || (cfg->line_search != 0 && cfg->line_search != 1) || (cfg->losses_ring && cfg->ring_len < 1))
        return pinn_fail_message(PINN_E_INVALID, "pinn_lbfgs_advance: invalid settings");
    int64_t stage_bytes = 3 * padded(n_params) * (int64_t)sizeof(float);
    int stage_on = stage_bytes <= STAGE_MAX_BYTES;
    int smem = stage_on ? (int)stage_bytes : 0;
    if (smem > 48 * 1024) {                          // the limit is per device: raise it to the most staging takes, once
        static std::atomic<uint64_t> raised{0};
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return pinn_fail_message(PINN_E_CUDA, cudaGetErrorString(e));
        uint64_t bit = dev < 64 ? 1ull << dev : 0;
        if (!bit || !(raised.load() & bit)) {
            e = cudaFuncSetAttribute(lbfgs_advance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGE_MAX_BYTES);
            if (e != cudaSuccess) return pinn_fail_message(PINN_E_CUDA, cudaGetErrorString(e));
            raised.fetch_or(bit);
        }
    }
    lbfgs_advance_kernel<<<1, THREADS, smem, (cudaStream_t)stream>>>(*cfg, n_params, params, grads_and_loss, state,
                                                                     status, stage_on);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return pinn_fail_message(PINN_E_CUDA, cudaGetErrorString(e));
    return PINN_OK;
}
