// wide_step_kernel (tensor-core tile kernel for wide networks) instantiations for NF = 2 first-order directions
#include "pinn_wide_kernel.cuh"

pinn::StepKernelFn pinn_wide_variant_nf2(int ns, int threads) {
    using namespace pinn::wide;
    if (threads == 512) {
        switch (ns) {
            case 0: return wide_step_kernel<2, 0, 512>;
            case 1: return wide_step_kernel<2, 1, 512>;
            case 2: return wide_step_kernel<2, 2, 512>;
            default: return nullptr;
        }
    }
    switch (ns) {
        case 0: return wide_step_kernel<2, 0, 256>;
        case 1: return wide_step_kernel<2, 1, 256>;
        case 2: return wide_step_kernel<2, 2, 256>;
        default: return nullptr;
    }
}
