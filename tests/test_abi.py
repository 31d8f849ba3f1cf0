""" The C-ABI library loads and exports every symbol include/pinn_b200.h declares (no compute calls:
runs without a GPU), and the ctypes mirror of PinnSpec matches the C layout. """
import ctypes as C
import os
import re
import subprocess

import pytest

from pydens_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'pinn_b200.h')


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(pinn_[a-z_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    lib = _native.load()
    names = declared_functions()
    assert len(names) >= 11
    for name in names:
        assert hasattr(lib, name), name
    assert set(names) == set(_native.EXPORTS)
    assert lib.pinn_abi_version() == _native.ABI_VERSION


def test_struct_layout_matches_c(tmp_path):
    src = tmp_path / 'sz.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pinn_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(PinnSpec), sizeof(PinnInstr),'
                   ' sizeof(PinnColumn), sizeof(PinnPlanInfo), offsetof(PinnSpec, eq_prog), offsetof(PinnSpec, ic_out),'
                   ' offsetof(PinnSpec, n_slots), sizeof(PinnAdam), offsetof(PinnAdam, lr), offsetof(PinnAdam, losses_ring),'
                   ' offsetof(PinnPlanInfo, small_batch_points), offsetof(PinnSpec, order));return 0;}\n')
    exe = tmp_path / 'sz'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    S = _native.PinnSpec
    assert got == [C.sizeof(S), C.sizeof(_native.PinnInstr), C.sizeof(_native.PinnColumn),
                   C.sizeof(_native.PinnPlanInfo), S.eq_prog.offset, S.ic_out.offset, S.n_slots.offset,
                   C.sizeof(_native.PinnAdam), _native.PinnAdam.lr.offset, _native.PinnAdam.losses_ring.offset,
                   _native.PinnPlanInfo.small_batch_points.offset, S.order.offset]


def test_plan_create_rejects_bad_spec_without_gpu():
    lib = _native.load()
    spec = _native.PinnSpec()
    spec.abi_version = 999
    plan = C.c_void_p()
    rc = lib.pinn_plan_create(C.byref(spec), 0, C.byref(plan))
    assert rc == _native.E_INVALID
    assert b'abi_version' in lib.pinn_last_error()


def test_library_is_sm90a_and_stages_weights_with_tma():
    """ The shipped .so holds sm_90a SASS whose step kernel stages the parameters with a TMA bulk copy
    (cp.async.bulk -> SASS UBLKCP) tracked by an mbarrier (SYNCS.*), and reduces with SHFL butterflies. """
    import shutil
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    fn = '_ZN4pinn11step_kernelILi2ELi2ELb0ELi256ELi16ELb0EEEvNS_7DevPlanENS_8StepArgsE'
    out = subprocess.run([cuobjdump, '-sass', '-fun', fn, _native.LIB_PATH], capture_output=True, text=True).stdout
    assert 'sm_90a' in out or 'SM90' in out.upper() or 'EF_CUDA_SM90' in out, out[:300]
    assert 'UBLKCP' in out                                  # TMA bulk copy global -> shared
    assert 'SYNCS' in out                                   # mbarrier expect_tx / try_wait
    assert out.count('SHFL.BFLY') >= 31                     # transposing butterfly of the gradient reduction
    assert 'LDS.128' in out                                 # broadcast 128-bit weight loads


def test_kernel_table_points_every_entry_at_its_kernel_instantiation():
    """ The kernel instantiations live in many build units that fill one table at load time; its lookup
    pinn::kernels(nf, ns, order) must hand out exactly step_kernel<NF, NS, GMEM, MAXT, 16, GEN> and the
    multi-step, small-batch, tile (64- and 128-wide) and coupled-system kernels of every (NF, NS), the five / six
    direction kernels and hi_step_kernel<NF, K> of orders 3 / 4, null where a jet set has no such kernel, and nothing
    for keys outside those.  Checked on the host against the exported kernel stubs — no GPU needed. """
    lib = C.CDLL(_native.LIB_PATH)

    class KernelSet(C.Structure):
        _fields_ = [('step', (C.c_void_p * 2) * 2), ('multi', C.c_void_p), ('small', C.c_void_p),
                    ('wide', C.c_void_p), ('maxt', C.c_int), ('wide128', C.c_void_p),
                    ('coupled', C.c_void_p * 2), ('coupled_wide128', C.c_void_p)]

    kernels = lib._ZN4pinn7kernelsEiii
    kernels.restype = C.POINTER(KernelSet)
    kernels.argtypes = [C.c_int, C.c_int, C.c_int]

    def addr(name):
        return C.cast(getattr(lib, name), C.c_void_p).value

    def step(nf, ns, gmem, maxt, gen):
        return addr('_ZN4pinn11step_kernelILi%dELi%dELb%dELi%dELi16ELb%dEEEvNS_7DevPlanENS_8StepArgsE' % (nf, ns, gmem, maxt, gen))

    def wide(name, nf, ns):
        return addr('_ZN4pinn4wide%d%sILi%dELi%dEEEvNS_7DevPlanENS_8StepArgsE' % (len(name), name, nf, ns))

    def tile_and_coupled_entries_are_null(k):
        return (k.wide, k.wide128, k.coupled[0], k.coupled[1], k.coupled_wide128) == (None,) * 5

    for nf in range(5):
        for ns in range(nf + 1):
            k = kernels(nf, ns, 2).contents
            maxt = 512 if 1 + nf + ns <= 3 else 256
            assert k.maxt == maxt
            for gen in (0, 1):
                assert [k.step[gen][0], k.step[gen][1]] == [step(nf, ns, 0, maxt, gen), step(nf, ns, 1, maxt, gen)], (nf, ns, gen)
            assert k.multi == addr('_ZN4pinn17multi_step_kernelILi%dELi%dELi%dELi16EEEvNS_7DevPlanENS_9MultiArgsE' % (nf, ns, maxt))
            assert k.small == addr('_ZN4pinn5small17small_step_kernelILi%dELi%dEEEvNS_7DevPlanENS_9MultiArgsE' % (nf, ns))
            assert k.wide == wide('wide_step_kernel', nf, ns), (nf, ns)
            assert k.wide128 == wide('wide128_step_kernel', nf, ns), (nf, ns)
            assert list(k.coupled) == [addr('_ZN4pinn19coupled_step_kernelILi%dELi%dELb%dELi%dEEEvNS_7DevPlanENS_8StepArgsE'
                                            % (nf, ns, gmem, maxt)) for gmem in (0, 1)], (nf, ns)
            assert k.coupled_wide128 == wide('wide128_coupled_step_kernel', nf, ns), (nf, ns)
        for order in (3, 4):
            k = kernels(nf, 0, order)
            if nf == 0:
                assert not k
                continue
            k = k.contents
            assert k.step[1][1] == addr('_ZN4pinn2hi14hi_step_kernelILi%dELi%dEEEvNS_7DevPlanENS_8StepArgsE' % (nf, order))
            assert (k.step[0][0], k.step[0][1], k.step[1][0], k.multi, k.small, k.maxt) == (None, None, None, None, None, 256)
            assert tile_and_coupled_entries_are_null(k), (nf, order)
            assert not kernels(nf, 1, order)
    for nf in (5, 6):
        k = kernels(nf, nf, 2).contents
        assert k.step[1][1] == step(nf, nf, 1, 256, 1) and k.maxt == 256
        assert (k.step[0][0], k.step[0][1], k.step[1][0], k.multi, k.small) == (None, None, None, None, None)
        assert tile_and_coupled_entries_are_null(k), nf
        for ns in range(nf):
            assert not kernels(nf, ns, 2)
        assert not kernels(nf, 0, 3) and not kernels(nf, 0, 4)
    for key in [(0, 1, 2), (4, 5, 2), (4, -1, 2), (-1, 0, 2), (7, 7, 2), (2, 0, 1), (2, 0, 5), (1, 0, 0)]:
        assert not kernels(*key), key
