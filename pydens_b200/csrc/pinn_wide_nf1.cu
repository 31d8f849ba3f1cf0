// wide_step_kernel (tensor-core tile kernel for wide networks) instantiations for NF = 1 first-order directions
#include "pinn_wide_kernel.cuh"

pinn::StepKernelFn pinn_wide_variant_nf1(int ns, int threads) {
    using namespace pinn::wide;
    if (threads == 512) {
        switch (ns) {
            case 0: return wide_step_kernel<1, 0, 512>;
            case 1: return wide_step_kernel<1, 1, 512>;
            default: return nullptr;
        }
    }
    switch (ns) {
        case 0: return wide_step_kernel<1, 0, 256>;
        case 1: return wide_step_kernel<1, 1, 256>;
        default: return nullptr;
    }
}
