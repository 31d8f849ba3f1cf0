""" ctypes binding of the C ABI in include/pinn_b200.h (libpinn_b200.so).

The library is the product's only compute path: if it is missing or does not export the ABI this
module raises — there is no CPU or eager fallback behind it.
"""
import ctypes as C
import os

ABI_VERSION = 11
MAX_LAYERS, MAX_DIMS, MAX_DIRS, MAX_VARS, MAX_PROG, MAX_SLOTS = 16, 8, 6, 4, 192, 96

ACT = {'none': 0, 'tanh': 1, 'sigmoid': 2, 'sin': 3, 'softplus': 4, 'silu': 5, 'gelu': 6}
COL_UNIFORM, COL_NORMAL, COL_CONST, COL_MIXTURE, COL_TNORMAL = 0, 1, 2, 3, 4
MAX_MIX = 4

E_INVALID, E_UNSUPPORTED, E_CUDA, E_ALIGN, E_WORKSPACE = -1, -2, -3, -4, -5


class PinnInstr(C.Structure):
    _fields_ = [('op', C.c_uint8), ('dst', C.c_uint8), ('a', C.c_uint8), ('b', C.c_uint8), ('imm', C.c_float)]


class PinnColumn(C.Structure):
    _fields_ = [('kind', C.c_int32), ('a', C.c_float), ('b', C.c_float),
                ('group', C.c_int32), ('n_comp', C.c_int32), ('cum_w', C.c_float * MAX_MIX),
                ('comp_kind', C.c_int32 * MAX_MIX), ('comp_a', C.c_float * MAX_MIX), ('comp_b', C.c_float * MAX_MIX)]


class PinnSpec(C.Structure):
    _fields_ = [
        ('abi_version', C.c_int32),
        ('n_layers', C.c_int32),
        ('widths', C.c_int32 * (MAX_LAYERS + 1)),
        ('act', C.c_int32 * MAX_LAYERS),
        ('skip_src', C.c_int32 * MAX_LAYERS),
        ('w_off', C.c_int32 * MAX_LAYERS),
        ('b_off', C.c_int32 * MAX_LAYERS),
        ('n_params', C.c_int32),
        ('log_scale_off', C.c_int32),
        ('n_vars', C.c_int32),
        ('var_off', C.c_int32 * MAX_VARS),
        ('ndims', C.c_int32), ('nparams', C.c_int32),
        ('has_bc', C.c_int32), ('has_ic', C.c_int32),
        ('bc_value', C.c_float),
        ('dom_lo', C.c_float * MAX_DIMS), ('dom_hi', C.c_float * MAX_DIMS),
        ('nf', C.c_int32), ('ns', C.c_int32),
        ('dir_col', C.c_int32 * MAX_DIRS),
        ('dir_vec', (C.c_float * MAX_DIMS) * MAX_DIRS),
        ('n_eq', C.c_int32),
        ('eq_prog', PinnInstr * MAX_PROG),
        ('eq_out', C.c_int32 * (1 + 1 + 2 * MAX_DIRS + MAX_VARS)),
        ('n_ic', C.c_int32),
        ('ic_prog', PinnInstr * MAX_PROG),
        ('ic_out', C.c_int32 * ((1 + 2 * MAX_DIRS) * (1 + MAX_VARS))),
        ('ic_has_vars', C.c_int32),
        ('n_slots', C.c_int32),
        ('order', C.c_int32),
    ]


class PinnPlanInfo(C.Structure):
    _fields_ = [
        ('nf', C.c_int32), ('ns', C.c_int32), ('channels', C.c_int32),
        ('threads_per_cta', C.c_int32), ('ctas_per_sm', C.c_int32),
        ('activations_in_smem', C.c_int32), ('smem_bytes', C.c_int32),
        ('regs_per_thread', C.c_int32), ('sm_count', C.c_int32),
        ('rows_per_point', C.c_int32),
        ('flops_per_point', C.c_int64),
        ('bytes_per_point', C.c_int32),
        ('tensor_core', C.c_int32),
        ('small_batch_points', C.c_int32),
    ]


class PinnAdam(C.Structure):
    _fields_ = [
        ('exp_avg', C.c_void_p), ('exp_avg_sq', C.c_void_p), ('mask', C.c_void_p), ('step_tensors', C.c_void_p),
        ('n_step_tensors', C.c_int32),
        ('lr', C.c_float), ('beta1', C.c_float), ('beta2', C.c_float), ('eps', C.c_float), ('weight_decay', C.c_float),
        ('losses_ring', C.c_void_p), ('ring_len', C.c_int64),
    ]


EXPORTS = ('pinn_last_error', 'pinn_abi_version', 'pinn_plan_create', 'pinn_plan_destroy',
           'pinn_workspace_bytes', 'pinn_out_floats', 'pinn_step', 'pinn_forward', 'pinn_sample',
           'pinn_record_loss', 'pinn_plan_info', 'pinn_comm_create', 'pinn_comm_connect', 'pinn_comm_destroy',
           'pinn_step_allreduce', 'pinn_comm_status', 'pinn_pipe_create', 'pinn_pipe_destroy', 'pinn_pipe_buffer',
           'pinn_pipe_step', 'pinn_pipe_finish', 'pinn_pipe_wait', 'pinn_pipe_sync', 'pinn_multi_step',
           'pinn_multi_step_max_points', 'pinn_step_adam')

LIB_PATH = os.environ.get('PYDENS_B200_LIB') or os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libpinn_b200.so')
_lib = None


class NativeError(RuntimeError):
    def __init__(self, code, message):
        super().__init__('libpinn_b200: %s (code %d)' % (message, code))
        self.code = code


class LibraryMissing(RuntimeError):
    """ libpinn_b200.so is absent or was built from another header. """


def load():
    """ Load libpinn_b200.so (once).  Raises RuntimeError if it is absent or its ABI does not match:
    the fused path has no fallback. """
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing('%s not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                           '(nvcc, sm_90a). pydens_b200 has no CPU fallback for the fit step.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise LibraryMissing('libpinn_b200.so does not export %s' % name)
    lib.pinn_last_error.restype = C.c_char_p
    lib.pinn_abi_version.restype = C.c_int
    lib.pinn_plan_create.argtypes = [C.POINTER(PinnSpec), C.c_int, C.POINTER(C.c_void_p)]
    lib.pinn_plan_destroy.argtypes = [C.c_void_p]
    lib.pinn_workspace_bytes.restype = C.c_size_t
    lib.pinn_workspace_bytes.argtypes = [C.c_void_p, C.c_int64]
    lib.pinn_out_floats.argtypes = [C.c_void_p]
    lib.pinn_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PinnColumn), C.c_uint64, C.c_void_p,
                              C.c_uint64, C.c_uint64, C.c_int64, C.c_float, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_size_t, C.c_void_p]
    lib.pinn_step_allreduce.argtypes = [C.c_void_p] + lib.pinn_step.argtypes
    lib.pinn_step_adam.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PinnColumn), C.c_uint64,
                                   C.c_void_p, C.c_uint64, C.c_int64, C.c_float, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_size_t, C.POINTER(PinnAdam), C.c_void_p]
    lib.pinn_comm_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_void_p]
    lib.pinn_comm_connect.argtypes = [C.c_void_p, C.c_char_p]
    lib.pinn_comm_destroy.argtypes = [C.c_void_p]
    lib.pinn_comm_status.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int]
    lib.pinn_pipe_create.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_void_p)]
    lib.pinn_pipe_destroy.argtypes = [C.c_void_p]
    lib.pinn_pipe_buffer.restype = C.c_void_p
    lib.pinn_pipe_buffer.argtypes = [C.c_void_p, C.c_int]
    lib.pinn_pipe_step.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.pinn_pipe_finish.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.pinn_pipe_wait.argtypes = [C.c_void_p, C.c_int]
    lib.pinn_pipe_sync.argtypes = [C.c_void_p]
    lib.pinn_multi_step_max_points.argtypes = [C.c_void_p]
    lib.pinn_multi_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_void_p, C.POINTER(PinnColumn), C.c_uint64, C.c_void_p, C.c_int64, C.c_int,
                                    C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                    C.c_void_p, C.c_int64, C.c_void_p]
    lib.pinn_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                 C.c_size_t, C.c_void_p]
    lib.pinn_sample.argtypes = [C.c_void_p, C.POINTER(PinnColumn), C.c_uint64, C.c_void_p, C.c_uint64,
                                C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p]
    lib.pinn_record_loss.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.pinn_plan_info.argtypes = [C.c_void_p, C.POINTER(PinnPlanInfo)]
    if lib.pinn_abi_version() != ABI_VERSION:
        raise LibraryMissing('libpinn_b200.so ABI %d != binding ABI %d: rebuild' % (lib.pinn_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise NativeError(rc, load().pinn_last_error().decode('utf-8', 'replace'))


def make_columns(cols, total):
    """ cols: per point column either (kind, a, b) or ('mix', group_key, [(weight, kind, a, b), ...]) — columns
    with the same group_key share the component draw — -> ctypes array, or None for the default U[0,1). """
    if cols is None:
        return None
    if isinstance(cols, PinnColumn * MAX_DIMS):           # already built
        return cols
    arr = (PinnColumn * MAX_DIMS)()
    groups = {}
    for i in range(MAX_DIMS):
        col = cols[i] if i < total else (COL_UNIFORM, 0.0, 1.0)
        if col[0] == 'mix':
            _, key, comps = col
            if not 2 <= len(comps) <= MAX_MIX:
                raise ValueError('a mixture column takes 2..%d components' % MAX_MIX)
            arr[i].kind = COL_MIXTURE
            arr[i].group = groups.setdefault(key, len(groups))
            arr[i].n_comp = len(comps)
            total_w, acc = float(sum(c[0] for c in comps)), 0.0
            for j, (w, kind, a, b) in enumerate(comps):
                acc += float(w)
                arr[i].cum_w[j] = 1.0 if j == len(comps) - 1 else acc / total_w
                arr[i].comp_kind[j], arr[i].comp_a[j], arr[i].comp_b[j] = int(kind), float(a), float(b)
        elif len(col) == 5:                               # (COL_TNORMAL, loc, scale, low, high)
            arr[i].kind, arr[i].a, arr[i].b = col[:3]
            arr[i].comp_a[0], arr[i].comp_b[0] = float(col[3]), float(col[4])
        else:
            arr[i].kind, arr[i].a, arr[i].b = col
    return arr


def build_spec(widths, acts, ndims, nparams, has_bc, bc_value, has_ic, domain, traced, var_offsets=None,
               w_off=None, b_off=None, log_scale_off=None, n_params=None, skips=None):
    """ Assemble a PinnSpec.

    widths: [total, n_1, ..., 1]; acts: activation name per linear layer ('none' for the last);
    domain: list of (lo, hi) per variable; traced: tracer.TracedEquation.
    Offsets default to the canonical flat layout W_0, b_0, W_1, b_1, ..., log_scale, V_0.. (padded to 4).
    """
    n_layers = len(widths) - 1
    if n_layers > MAX_LAYERS:
        raise ValueError('too many layers')
    s = PinnSpec()
    s.abi_version = ABI_VERSION
    s.n_layers = n_layers
    off = 0
    for l in range(n_layers):
        s.widths[l] = widths[l]
        s.act[l] = ACT[acts[l]]
        s.skip_src[l] = -1 if not skips or skips[l] is None else int(skips[l])
        if w_off is None:
            s.w_off[l] = off
            off += widths[l] * widths[l + 1]
            s.b_off[l] = off
            off += widths[l + 1]
        else:
            s.w_off[l], s.b_off[l] = w_off[l], b_off[l]
    s.widths[n_layers] = widths[n_layers]
    if log_scale_off is None:
        log_scale_off = off
        off += 1
    s.log_scale_off = log_scale_off
    names = traced.var_names
    s.n_vars = len(names)
    for i, name in enumerate(names):
        if var_offsets is None:
            s.var_off[i] = off
            off += 1
        else:
            s.var_off[i] = var_offsets[name]
    s.n_params = n_params if n_params is not None else (off + 3) // 4 * 4
    s.ndims, s.nparams = ndims, nparams
    s.has_bc, s.has_ic = int(bool(has_bc)), int(bool(has_ic))
    s.bc_value = float(bc_value) if has_bc else 0.0
    for i in range(ndims):
        s.dom_lo[i], s.dom_hi[i] = float(domain[i][0]), float(domain[i][1])
    s.nf, s.ns = traced.nf, traced.ns
    s.order = int(getattr(traced, 'order', 2)) if getattr(traced, 'order', 2) > 2 else 0
    for d, vec in enumerate(traced.dir_vecs):
        s.dir_col[d] = traced.dirs[d]
        for k, v in enumerate(vec):
            s.dir_vec[d][k] = float(v)
    fill_program(s.eq_prog, traced.eq_prog)
    s.n_eq = len(traced.eq_prog)
    for i, slot in enumerate(traced.eq_prog.outs):
        s.eq_out[i] = slot
    if has_ic:
        fill_program(s.ic_prog, traced.ic_prog)
        s.n_ic = len(traced.ic_prog)
        for i, slot in enumerate(traced.ic_prog.outs):
            s.ic_out[i] = slot
        s.ic_has_vars = int(traced.ic_has_vars)
    s.n_slots = max(traced.n_slots, traced.channels)
    return s


def fill_program(dst, prog):
    for i, (op, d, a, b, imm) in enumerate(prog.instrs):
        dst[i].op, dst[i].dst, dst[i].a, dst[i].b, dst[i].imm = op, d, a, b, imm
