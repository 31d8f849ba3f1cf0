""" What every plan launches: the placement, the workspace and the bits of one call of each entry point.

For every problem of the tests' registries (tests/problems*.py) and every placement override plan creation reads, this
records the plan-creation return code, every PinnPlanInfo field, pinn_workspace_bytes, pinn_out_floats and
pinn_multi_step_max_points, and the SHA-256 digests of what one call of each entry point writes:
  * pinn_step at n = 1000 in-kernel sampled points: [grads | loss] and the residual;
  * pinn_step_adam at n = 1000: the parameters after the update and [grads | loss];
  * pinn_forward at 257 explicit points;
  * where the persistent kernels exist: the parameters after pinn_multi_step_terms of 4 steps at n = 100 (the cluster
    kernel) and n = 300 (the multi-step kernel), and after a two-member pinn_multi_step_ensemble;
  * for the tile kernels, the two steps again with PINN_WIDE_CTAS=7 set after the plan exists.
The kernels' sums run in a fixed order, so the digests pin down the kernel, the grid, the block and the shared memory
each launch uses.  tests/test_gpu_plan_records.py compares a build against tests/golden/plan_records.json, which

    python tools/plan_records.py tests/golden/plan_records.json

writes (on the device the fixture names: the placement depends on its SM count and shared memory).
"""
import contextlib
import ctypes as C
import hashlib
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

import problems as P                                    # noqa: E402
import problems_coupled as PC                           # noqa: E402
import problems_systems as PS                           # noqa: E402
import problems_wide as PW                              # noqa: E402
import problems_wide_coupled as PWC                     # noqa: E402

REGISTRIES = {'problems': P.PROBLEMS, 'systems': PS.PROBLEMS, 'coupled': PC.PROBLEMS, 'wide': PW.PROBLEMS,
              'wide_coupled': PWC.PROBLEMS}
OVERRIDES = {
    'default': {},
    'smem': {'PINN_FORCE_MODE': 'smem'},
    'gmem': {'PINN_FORCE_MODE': 'gmem'},
    'gmem_w1': {'PINN_FORCE_MODE': 'gmem', 'PINN_GMEM_WARPS': '1'},
    'thread': {'PINN_FORCE_KERNEL': 'thread'},
    'wide': {'PINN_FORCE_KERNEL': 'wide'},
    'wide128': {'PINN_FORCE_KERNEL': 'wide128'},
}
N_STEP, N_FORWARD, SEED = 1000, 257, 2024


def names():
    return ['%s/%s' % (reg, n) for reg, problems in REGISTRIES.items() for n in problems]


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def device():
    import torch
    prop = torch.cuda.get_device_properties(0)
    return dict(name=prop.name, sm_count=prop.multi_processor_count, smem_optin=prop.shared_memory_per_block_optin)


def spec_and_params(name):
    """ -> (PinnSpec, initial flat parameters) of a registry problem, from a fused Solver's engine """
    import torch
    from pydens_b200 import Solver, D, V, _native as N
    reg, key = name.split('/')
    cfg = REGISTRIES[reg][key]
    pkg_V = lambda n, init: V(n, data=torch.Tensor([init]))    # noqa: E731
    eq = cfg['equation']
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)            # systems: the [N, m] vs [N, 1] broadcast of the trial run
        solver = Solver(lambda u, *xs: eq(u, *xs, D=D, V=pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                        initial_condition=cfg['ic_factory'](pkg_V) if 'ic_factory' in cfg else cfg['ic'],
                        boundary_condition=cfg['bc'], domain=cfg['domain'], layout=cfg['layout'],
                        features=cfg['features'], activation=cfg['activation'], device='cuda', backend='fused',
                        seed=1234)
    if 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    eng = solver._get_engine()
    return N.PinnSpec.from_buffer_copy(eng.spec), eng.flat.detach().cpu().numpy().copy()


def _digest(*tensors):
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().cpu().numpy().tobytes())
    return h.hexdigest()


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _steps(lib, plan, spec, params, ws, stream):
    """ one sampled pinn_step and one pinn_step_adam: their return codes and digests """
    import torch
    from pydens_b200 import _native as N
    dev, n_out = params.device, spec.n_params + 4
    out = torch.zeros(n_out, device=dev)
    res = torch.zeros(N_STEP, device=dev)
    rc = lib.pinn_step(plan, _ptr(params), None, None, C.c_uint64(SEED), None, C.c_uint64(5), C.c_uint64(0),
                       C.c_int64(N_STEP), C.c_float(1.0 / N_STEP), _ptr(out), _ptr(res), _ptr(ws),
                       C.c_size_t(ws.numel()), stream)
    torch.cuda.synchronize()
    r = dict(step_rc=rc, step=_digest(out, res) if rc == 0 else None)
    p = params.clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    mask, steps = torch.ones_like(p), torch.zeros(4, device=dev)
    counter, ring = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(8, device=dev)
    out.zero_()
    adam = N.PinnAdam(m.data_ptr(), v.data_ptr(), mask.data_ptr(), steps.data_ptr(), 4, 1e-3, 0.9, 0.999, 1e-8, 0.01,
                      ring.data_ptr(), ring.numel())
    rc = lib.pinn_step_adam(plan, None, _ptr(p), None, None, C.c_uint64(SEED), _ptr(counter), C.c_uint64(0),
                            C.c_int64(N_STEP), C.c_float(1.0 / N_STEP), _ptr(out), None, _ptr(ws),
                            C.c_size_t(ws.numel()), C.byref(adam), stream)
    torch.cuda.synchronize()
    r.update(adam_rc=rc, adam=_digest(p, out) if rc == 0 else None)
    return r


def _persistent(lib, plan, spec, params, stream):
    """ pinn_multi_step_terms at 100 and 300 points and a two-member pinn_multi_step_ensemble """
    import torch
    from pydens_b200 import _native as N
    dev, r = params.device, {}

    def state():
        return dict(p=params.clone(), m=torch.zeros_like(params), v=torch.zeros_like(params),
                    mask=torch.ones_like(params), steps=torch.zeros(4, device=dev),
                    counter=torch.zeros(1, dtype=torch.int64, device=dev), ring=torch.zeros(64, device=dev))

    for n in (100, 300):
        s = state()
        rc = lib.pinn_multi_step_terms(plan, _ptr(s['p']), _ptr(s['m']), _ptr(s['v']), _ptr(s['mask']),
                                       _ptr(s['steps']), C.c_int(4), None, None, C.c_uint64(SEED), _ptr(s['counter']),
                                       C.c_int64(n), C.c_int(4), C.c_float(0.01), C.c_float(0.9), C.c_float(0.999),
                                       C.c_float(1e-8), C.c_float(0.0), C.c_float(0.0), _ptr(s['ring']),
                                       C.c_int64(64), C.c_float(1.0 / n), C.c_int(0), None, stream)
        torch.cuda.synchronize()
        r['multi%d_rc' % n], r['multi%d' % n] = rc, _digest(s['p'], s['ring']) if rc == 0 else None
    members = [state() for _ in range(2)]
    table = (N.PinnMember * 2)()
    for j, s in enumerate(members):
        t = table[j]
        t.params, t.exp_avg, t.exp_avg_sq, t.mask = (s['p'].data_ptr(), s['m'].data_ptr(), s['v'].data_ptr(),
                                                     s['mask'].data_ptr())
        t.step_tensors, t.n_step_tensors, t.opt_step0 = s['steps'].data_ptr(), 4, 0.0
        t.points, t.seed, t.step_counter, t.losses_ring = None, SEED + j, s['counter'].data_ptr(), s['ring'].data_ptr()
    rc = lib.pinn_multi_step_ensemble(plan, 2, table, C.c_int64(100), C.c_int(4), C.c_float(0.01), C.c_float(0.9),
                                      C.c_float(0.999), C.c_float(1e-8), C.c_float(0.0), C.c_int64(64),
                                      C.c_float(0.01), C.c_int(0), None, None, stream)
    torch.cuda.synchronize()
    r['ensemble_rc'] = rc
    r['ensemble'] = _digest(*[s[k] for s in members for k in ('p', 'ring')]) if rc == 0 else None
    return r


def record(spec, flat, overrides):
    """ the record of one plan, created under `overrides` """
    import torch
    from pydens_b200 import _native as N
    lib, dev = N.load(), torch.device('cuda:0')
    plan = C.c_void_p()
    with env(**overrides):
        rc = lib.pinn_plan_create(C.byref(spec), 0, C.byref(plan))
    if rc != 0:
        return dict(create_rc=rc)
    try:
        info = N.PinnPlanInfo()
        N.check(lib.pinn_plan_info(plan, C.byref(info)))
        r = dict(create_rc=0, info={f: getattr(info, f) for f, _ in N.PinnPlanInfo._fields_},
                 workspace_bytes=lib.pinn_workspace_bytes(plan, N_STEP), out_floats=lib.pinn_out_floats(plan),
                 multi_step_max_points=lib.pinn_multi_step_max_points(plan))
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        params = torch.from_numpy(flat).to(dev)
        ws = torch.zeros(r['workspace_bytes'], dtype=torch.uint8, device=dev)
        r.update(_steps(lib, plan, spec, params, ws, stream))
        k = spec.widths[spec.n_layers]
        rng = np.random.RandomState(SEED)
        pts = torch.from_numpy(rng.uniform(0.0, 1.0, size=(N_FORWARD, spec.ndims + spec.nparams)).astype(np.float32)).to(dev)
        u = torch.zeros(N_FORWARD * k, device=dev)
        rc = lib.pinn_forward(plan, _ptr(params), _ptr(pts), C.c_int64(N_FORWARD), _ptr(u), _ptr(ws),
                              C.c_size_t(ws.numel()), stream)
        torch.cuda.synchronize()
        r.update(forward_rc=rc, forward=_digest(u) if rc == 0 else None)
        if r['multi_step_max_points'] > 0:
            r.update(_persistent(lib, plan, spec, params, stream))
        if info.tensor_core:
            with env(PINN_WIDE_CTAS='7'):
                r['wide_ctas7'] = _steps(lib, plan, spec, params, ws, stream)
        return r
    finally:
        lib.pinn_plan_destroy(plan)


def problem_records(name):
    spec, flat = spec_and_params(name)
    return {o: record(spec, flat, kv) for o, kv in OVERRIDES.items()}


def main(path):
    fixture = dict(device=device(), records={name: problem_records(name) for name in names()})
    with open(path, 'w') as f:
        json.dump(fixture, f, indent=1, sort_keys=True)
        f.write('\n')
    print('%d problems x %d overrides -> %s' % (len(fixture['records']), len(OVERRIDES), path))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden', 'plan_records.json'))
