// pinn_instances.cu — the kernel instantiations of one build unit.  __graft_entry__.py compiles this file once per
// entry of its unit table (UNITS), with the unit's kernel family PINN_UNIT, its direction count PINN_NF and the range
// PINN_LO..PINN_HI of NS (of the derivative order for PINN_HI_JET) as -D flags, so that the heavy instantiations
// compile in parallel.  Each unit enters its kernels into the table of pinn_kernels.cu during static initialisation.
#include <utility>

#define PINN_STEP 1          // step_kernel, plain problems
#define PINN_STEP_GEN 2      // step_kernel, general problems, and the persistent multi-step kernel
#define PINN_STEP_GMEM 3     // five / six directions: the general step_kernel with per-point state in global memory
#define PINN_HI_JET 4        // hi_step_kernel, derivatives of order 3 / 4
#define PINN_WIDE 5          // wide_step_kernel, the tensor-core tile kernel
#define PINN_SMALL 6         // small_step_kernel, the tiny-batch cluster kernel
#define PINN_WIDE128 7       // wide_step_kernel of the 128-wide class

#if PINN_UNIT == PINN_HI_JET
#include "pinn_hi_kernel.cuh"
#elif PINN_UNIT == PINN_WIDE || PINN_UNIT == PINN_WIDE128
#include "pinn_wide_kernel.cuh"
#elif PINN_UNIT == PINN_SMALL
#include "pinn_small_kernel.cuh"
#else
#include "pinn_step_kernel.cuh"
#endif

namespace pinn {
namespace {

constexpr int NF = PINN_NF;

template <int J>
void enter() {
#if PINN_UNIT == PINN_STEP || PINN_UNIT == PINN_STEP_GEN
    constexpr bool GEN = PINN_UNIT == PINN_STEP_GEN;
    using Cfg = VariantCfg<NF, J>;
    KernelSet& k = kernel_slot(NF, J, 2);
    k.step[GEN][0] = step_kernel<NF, J, false, Cfg::MAXT, Cfg::JF, GEN>;
    k.step[GEN][1] = step_kernel<NF, J, true, Cfg::MAXT, Cfg::JF, GEN>;
    if constexpr (GEN) k.multi = multi_step_kernel<NF, J, Cfg::MAXT, Cfg::JF>;
    k.maxt = Cfg::MAXT;
#elif PINN_UNIT == PINN_STEP_GMEM
    // 13 jet channels per unit do not fit shared memory for any network worth the name; the tracer promotes every
    // direction of such a problem to second order, so NS = NF is the only combination that occurs
    static_assert(J == NF, "five / six directions: NS = NF only");
    using Cfg = VariantCfg<NF, NF>;
    KernelSet& k = kernel_slot(NF, NF, 2);
    k.step[1][1] = step_kernel<NF, NF, true, Cfg::MAXT, Cfg::JF, true>;
    k.maxt = Cfg::MAXT;
#elif PINN_UNIT == PINN_HI_JET
    KernelSet& k = kernel_slot(NF, 0, J);
    k.step[1][1] = hi::hi_step_kernel<NF, J>;
    k.maxt = 256;
#elif PINN_UNIT == PINN_WIDE
    KernelSet& k = kernel_slot(NF, J, 2);
    k.wide[0] = wide::wide_step_kernel<NF, J, 512>;
    k.wide[1] = wide::wide_step_kernel<NF, J, 256>;
#elif PINN_UNIT == PINN_WIDE128
    kernel_slot(NF, J, 2).wide128 = wide::wide128_step_kernel<NF, J>;
#elif PINN_UNIT == PINN_SMALL
    kernel_slot(NF, J, 2).small = small::small_step_kernel<NF, J>;
#else
#error "PINN_UNIT names no kernel family"
#endif
}

template <int... I>
bool enter_all(std::integer_sequence<int, I...>) {
    (enter<PINN_LO + I>(), ...);
    return true;
}

const bool entered = enter_all(std::make_integer_sequence<int, PINN_HI - PINN_LO + 1>());

}  // namespace
}  // namespace pinn
