// wide_step_kernel (tensor-core tile kernel for wide networks) instantiations for NF = 0 first-order directions
#include "pinn_wide_kernel.cuh"

pinn::StepKernelFn pinn_wide_variant_nf0(int ns, int threads) {
    using namespace pinn::wide;
    if (threads == 512) {
        switch (ns) {
            case 0: return wide_step_kernel<0, 0, 512>;

            default: return nullptr;
        }
    }
    switch (ns) {
        case 0: return wide_step_kernel<0, 0, 256>;

        default: return nullptr;
    }
}
