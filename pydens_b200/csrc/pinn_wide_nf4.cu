// wide_step_kernel (tensor-core tile kernel for wide networks) instantiations for NF = 4 first-order directions
#include "pinn_wide_kernel.cuh"

pinn::StepKernelFn pinn_wide_variant_nf4(int ns, int threads) {
    using namespace pinn::wide;
    if (threads == 512) {
        switch (ns) {
            case 0: return wide_step_kernel<4, 0, 512>;
            case 1: return wide_step_kernel<4, 1, 512>;
            case 2: return wide_step_kernel<4, 2, 512>;
            case 3: return wide_step_kernel<4, 3, 512>;
            case 4: return wide_step_kernel<4, 4, 512>;
            default: return nullptr;
        }
    }
    switch (ns) {
        case 0: return wide_step_kernel<4, 0, 256>;
        case 1: return wide_step_kernel<4, 1, 256>;
        case 2: return wide_step_kernel<4, 2, 256>;
        case 3: return wide_step_kernel<4, 3, 256>;
        case 4: return wide_step_kernel<4, 4, 256>;
        default: return nullptr;
    }
}
