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


def test_variant_tables_point_at_the_right_kernel_instantiations():
    """ The step_kernel instantiations live in several translation units (one per NF, the heavy general ones split
    by NS); the host dispatch tables must hand out exactly step_kernel<NF, NS, GMEM, MAXT, 16, GEN> for every
    (NF, NS).  Checked on the host against the exported kernel stubs — no GPU needed. """
    import ctypes as C
    lib = C.CDLL(_native.LIB_PATH)

    class Variant(C.Structure):
        _fields_ = [('nf', C.c_int), ('ns', C.c_int), ('smem_fn', C.c_void_p), ('gmem_fn', C.c_void_p),
                    ('smem_gen_fn', C.c_void_p), ('gmem_gen_fn', C.c_void_p), ('multi_fn', C.c_void_p), ('maxt', C.c_int)]

    def stub(nf, ns, gmem, maxt, gen):
        name = '_ZN4pinn11step_kernelILi%dELi%dELb%dELi%dELi16ELb%dEEEvNS_7DevPlanENS_8StepArgsE' % (nf, ns, gmem, maxt, gen)
        return C.cast(getattr(lib, name), C.c_void_p).value

    for nf in range(5):
        for gen in (0, 1):
            fn = getattr(lib, '_Z%dpinn_variants_%snf%di' % (17 if not gen else 21, 'gen_' if gen else '', nf))
            fn.restype = C.POINTER(Variant)
            fn.argtypes = [C.c_int]
            for ns in range(nf + 1):
                v = fn(ns).contents
                maxt = 512 if 1 + nf + ns <= 3 else 256
                assert (v.nf, v.ns, v.maxt) == (nf, ns, maxt)
                smem, gmem = (v.smem_gen_fn, v.gmem_gen_fn) if gen else (v.smem_fn, v.gmem_fn)
                assert smem == stub(nf, ns, 0, maxt, gen) and gmem == stub(nf, ns, 1, maxt, gen), (nf, ns, gen)
                other = (v.smem_fn, v.gmem_fn) if gen else (v.smem_gen_fn, v.gmem_gen_fn)
                assert other == (None, None)           # the sibling unit fills the other half (merged at plan creation)
                # the persistent multi-step kernel rides in the general half
                mname = '_ZN4pinn17multi_step_kernelILi%dELi%dELi%dELi16EEEvNS_7DevPlanENS_9MultiArgsE' % (nf, ns, maxt)
                assert v.multi_fn == (C.cast(getattr(lib, mname), C.c_void_p).value if gen else None)
            assert not fn(nf + 1) and not fn(-1)
