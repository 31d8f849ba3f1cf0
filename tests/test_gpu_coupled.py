""" Coupled systems (networks with 2..4 outputs) on the GPU, CPU twin: test_coupled.py.  coupled_step_kernel through the
bare C ABI at every jet set x k x placement against the fp64 oracle tensor by tensor, batch edges, the reference goldens
at every placement, Solver.fit against the reference's own fit with both Adam forms, predict [N, k], in-kernel sampling,
bit-reproducibility, graph replay, constraints added by autograd, tiny batches, two GPUs, and what the coupled kernels
refuse. """
import contextlib
import ctypes as C
import os
import warnings

import numpy as np
import pytest
import torch

import problems_coupled as PC
from helpers import load_golden, rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

if torch.cuda.is_available():
    from gpu_helpers import Replay
    from pydens_b200 import Solver, D, V
    from pydens_b200 import _native as N
    from test_coupled import coupled_spec, folded, crit_key, oracle_loss_and_grads, random_setup, tolerances

JET_SETS = [(nf, ns) for nf in range(5) for ns in range(nf + 1)]

PLACEMENTS = {'default': {}, 'gmem1': {'PINN_FORCE_MODE': 'gmem', 'PINN_GMEM_WARPS': '1'},
              'gmem3': {'PINN_FORCE_MODE': 'gmem', 'PINN_GMEM_WARPS': '3'}}


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


class Plan:
    """ A plan of the bare C ABI for one spec (placement from the environment at creation). """

    def __init__(self, spec, placement='default'):
        self.lib, self.spec = N.load(), spec
        self.dev = torch.device('cuda:0')
        self.plan = C.c_void_p()
        with env(**PLACEMENTS[placement]):
            N.check(self.lib.pinn_plan_create(C.byref(spec), 0, C.byref(self.plan)))
        self.info = N.PinnPlanInfo()
        N.check(self.lib.pinn_plan_info(self.plan, C.byref(self.info)))

    def __del__(self):
        if self.plan:
            self.lib.pinn_plan_destroy(self.plan)

    def step(self, params, points, inv_n=None):
        n, k = points.shape[0], self.spec.widths[self.spec.n_layers]
        flat = torch.from_numpy(np.ascontiguousarray(params, dtype=np.float32)).to(self.dev)
        pts = torch.from_numpy(np.ascontiguousarray(points, dtype=np.float32)).to(self.dev)
        out = torch.zeros(self.spec.n_params + 4, dtype=torch.float32, device=self.dev)
        res = torch.zeros(n, dtype=torch.float32, device=self.dev)
        u = torch.zeros((n, k), dtype=torch.float32, device=self.dev)
        ws = torch.zeros(self.lib.pinn_workspace_bytes(self.plan, n), dtype=torch.uint8, device=self.dev)
        stream = C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)
        N.check(self.lib.pinn_step(self.plan, C.c_void_p(flat.data_ptr()), C.c_void_p(pts.data_ptr()), None, C.c_uint64(0),
                                   None, C.c_uint64(0), C.c_uint64(0), C.c_int64(n), C.c_float(1.0 / n if inv_n is None else inv_n),
                                   C.c_void_p(out.data_ptr()), C.c_void_p(res.data_ptr()),
                                   C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel()), stream))
        N.check(self.lib.pinn_forward(self.plan, C.c_void_p(flat.data_ptr()), C.c_void_p(pts.data_ptr()), C.c_int64(n),
                                      C.c_void_p(u.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel()), stream))
        torch.cuda.synchronize(self.dev)
        o = out.cpu().numpy()
        return float(o[self.spec.n_params]), res.cpu().numpy(), o[:self.spec.n_params].copy(), u.cpu().numpy()


def check_tensors(spec, grads, ref, tol):
    """ every weight and bias, d/dlog_scale and every d/dV against the reference vector """
    for l in range(spec.n_layers):
        w = slice(spec.w_off[l], spec.w_off[l] + spec.widths[l] * spec.widths[l + 1])
        b = slice(spec.b_off[l], spec.b_off[l] + spec.widths[l + 1])
        assert rel_l2(grads[w], ref[w]) <= tol, 'W%d' % l
        assert rel_l2(grads[b], ref[b]) <= tol, 'b%d' % l
    scale = 1e-3 * np.abs(ref).max()
    for off in [spec.log_scale_off] + [spec.var_off[i] for i in range(spec.n_vars)]:
        assert abs(grads[off] - ref[off]) <= tol * max(abs(ref[off]), scale), off


# ------------------------------------------------------------------------------------------------------------------
# the C ABI against the fp64 oracle: every jet set x k x placement
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('placement', list(PLACEMENTS))
@pytest.mark.parametrize('k', [2, 3, 4])
@pytest.mark.parametrize('jet', JET_SETS, ids=['nf%d_ns%d' % j for j in JET_SETS])
def test_every_jet_set_and_output_count_matches_fp64_oracle(jet, k, placement):
    seed = 1000 + 17 * JET_SETS.index(jet) + k
    cfg, prob, params, pts, (key, crit, red, r64, thr), spec = random_setup(seed, k=k, jet=jet, kind='mse')
    plan = Plan(spec, placement)
    assert plan.info.tensor_core == 0 and plan.info.small_batch_points == 0
    if placement != 'default':
        assert plan.info.activations_in_smem == 0
        assert plan.info.threads_per_cta == 32 * int(PLACEMENTS[placement]['PINN_GMEM_WARPS'])
    loss, residual, grads, u = plan.step(params, pts)
    ref_loss, ref_res, ref_grads = oracle_loss_and_grads(prob, pts.astype(np.float64), criterion=crit)
    cond, _ = tolerances(cfg, r64, thr)
    assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), cfg['tag']
    assert rel_l2(residual, folded(ref_res, k)) <= 2e-5 * cond, cfg['tag']
    assert rel_l2(grads, ref_grads.numpy()) <= 1e-4 * cond, cfg['tag']
    check_tensors(spec, grads, ref_grads.numpy(), 2e-4 * cond)
    assert u.shape == (pts.shape[0], k) and rel_l2(u, prob.predict(pts.astype(np.float64)).reshape(-1, k)) <= 1e-5


@pytest.mark.parametrize('placement', list(PLACEMENTS))
def test_batch_edges_match_fp64_oracle(placement):
    cfg, prob, params, _, _, spec = random_setup(7, k=3, jet=(2, 2), kind='mse')
    plan = Plan(spec, placement)
    warps = plan.info.threads_per_cta // 32
    full = 32 * warps * plan.info.sm_count
    rng = np.random.RandomState(5)
    for n in (1, 33, full - 1, full + 1, 200003):
        ranges = list(cfg['domain']) + [(0.0, 1.0)] * cfg['nparams']
        pts = np.concatenate([rng.uniform(lo + 1e-3, hi - 1e-3, size=(n, 1)) for lo, hi in ranges], axis=1).astype(np.float32)
        loss, residual, grads, u = plan.step(params, pts)
        ref_loss, ref_res, ref_grads = oracle_loss_and_grads(prob, pts.astype(np.float64))
        r = np.asarray(ref_res).reshape(-1, 3)
        cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(r)))), 1e-30))
        assert abs(loss - ref_loss) <= 5e-5 * cond * abs(ref_loss), n
        assert rel_l2(residual, folded(ref_res, 3)) <= 2e-5 * cond, n
        assert rel_l2(grads, ref_grads.numpy()) <= 2e-4 * cond, n


# ------------------------------------------------------------------------------------------------------------------
# the reference goldens
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('placement', list(PLACEMENTS))
@pytest.mark.parametrize('name', list(PC.PROBLEMS))
def test_c_abi_matches_reference_golden(name, placement):
    g = load_golden(name)
    spec = coupled_spec(name)
    loss, residual, grads, u = Plan(spec, placement).step(g['params'], g['points'])
    assert abs(loss - float(g['loss'])) <= 1e-5 * abs(float(g['loss']))
    assert rel_l2(residual, folded(g['residual'], PC.PROBLEMS[name]['m'], crit_key(name))) <= 1e-5
    assert rel_l2(grads, g['grads']) <= 1e-4
    check_tensors(spec, grads, g['grads'], 1e-4)
    assert rel_l2(u, g['u']) <= 1e-5


def pkg_V(name, init):
    return V(name, data=torch.Tensor([init]))


def make_solver(name, backend='fused', **kw):
    cfg = PC.PROBLEMS[name]
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)           # the [N, m] vs [N, 1] broadcast of the throw-away run
        solver = Solver(PC.bind(name, D, pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                        initial_condition=PC.make_ic(name, pkg_V), boundary_condition=cfg['bc'], domain=cfg['domain'],
                        layout=cfg['layout'], features=cfg['features'], activation=cfg['activation'],
                        device='cuda', backend=backend, seed=1234, **kw)
    if 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


@pytest.mark.parametrize('name', list(PC.PROBLEMS))
def test_solver_matches_reference_golden_and_predicts_n_by_k(name):
    g = load_golden(name)
    solver = make_solver(name)
    solver.load_flat_params(g['params'])
    crit = PC.torch_criterion(name)
    assert solver._fused_possible(crit, ('equation',))[0]
    loss, grads, residual = solver.loss_and_grads(g['points'])
    assert abs(loss - float(g['loss'])) <= 1e-5 * abs(float(g['loss']))
    assert rel_l2(grads.cpu().numpy()[:g['grads'].size], g['grads']) <= 1e-4
    u = solver.predict(*[g['points'][:, i] for i in range(g['points'].shape[1])])
    assert isinstance(u, np.ndarray) and u.dtype == np.float32 and u.shape == g['u'].shape
    assert rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('fused_adam', ['1', '0'])
@pytest.mark.parametrize('name', list(PC.GOLDEN_TRAJ))
def test_fit_follows_the_reference_fit(name, fused_adam):
    """ The reference's own Solver.fit on the same batches: in-kernel Adam (pinn_step_adam) and torch's optimizer. """
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    solver = make_solver(name)
    solver.load_flat_params(g['params'])
    batches = [PC.make_points(name, batch, seed=1000 + i) for i in range(niters)]
    with env(PYDENS_B200_FUSED_ADAM=fused_adam), warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        solver.fit(niters=niters, batch_size=batch, sampler=Replay(batches), lr=lr, criterion=PC.torch_criterion(name))
    assert not [w for w in caught if 'pydens_b200' in str(w.message)]      # no autograd fallback, no notice
    losses, ref = np.asarray(solver.losses, dtype=np.float64), g['traj_losses'].astype(np.float64)
    assert np.max(np.abs(losses - ref) / np.abs(ref)) <= 2e-3
    flat = solver.flat_params().cpu().numpy()[:g['traj_params'].size]
    assert rel_l2(flat, g['traj_params']) <= 1e-3


# ------------------------------------------------------------------------------------------------------------------
# sampling, reproducibility, graphs
# ------------------------------------------------------------------------------------------------------------------
def test_in_kernel_sampling_equals_explicit_points_and_runs_are_bit_identical():
    solver = make_solver('navier_stokes2d')
    eng = solver._get_engine()
    n = 70001
    outs = []
    for _ in range(2):
        eng._step(None, None, n, 1.0 / n, 0, use_counter=False, step_value=5)
        torch.cuda.synchronize()
        outs.append(eng.out.clone())
    assert torch.equal(outs[0], outs[1])
    pts = eng.sample(n, step=5)
    eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
    torch.cuda.synchronize()
    assert torch.equal(eng.out, outs[0])


def test_graph_replay_equals_plain_launches():
    runs = []
    for no_graph in ('0', '1'):
        solver = make_solver('brusselator')
        with env(PYDENS_B200_NO_GRAPH=no_graph):
            solver.fit(niters=24, batch_size=5000, lr=0.01)
        runs.append((np.asarray(solver.losses), solver.flat_params().cpu().numpy()))
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
    again = make_solver('brusselator')
    again.fit(niters=24, batch_size=5000, lr=0.01)
    assert np.array_equal(np.asarray(again.losses), runs[0][0])


def test_repeated_fit_and_frozen_layers():
    solver = make_solver('lotka_volterra')
    solver.fit(niters=10, batch_size=2000, lr=0.01)
    lin0 = [m for m in solver.model.conv_block.modules() if isinstance(m, torch.nn.Linear)][0]
    lin0.weight.requires_grad_(False)
    lin0.bias.requires_grad_(False)
    w0, b0 = lin0.weight.detach().clone(), lin0.bias.detach().clone()
    solver.fit(niters=10, batch_size=2000, lr=0.01)
    assert solver._engine is not None and len(solver.losses) == 20 and np.isfinite(solver.losses[-1])
    assert torch.equal(lin0.weight.detach(), w0) and torch.equal(lin0.bias.detach(), b0)


# ------------------------------------------------------------------------------------------------------------------
# constraints, tiny batches, two GPUs
# ------------------------------------------------------------------------------------------------------------------
def test_constraint_is_added_by_autograd_on_top_of_the_fused_equation():
    name = 'navier_stokes2d'
    batches = [PC.make_points(name, 256, seed=2000 + i) for i in range(8)]
    cons = lambda u, x, y: u(torch.tensor([0.5]), torch.tensor([0.5]))[:, 2:3] - 0.1     # pin the pressure at a point
    curves = []
    for backend in ('fused', 'torch'):
        solver = make_solver(name, backend=backend, constraints=[cons])
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', UserWarning)
            solver.fit(niters=8, batch_size=256, sampler=Replay(list(batches)), lr=0.005,
                       loss_terms=['equation', 'constraint_0'])
        curves.append(np.asarray(solver.losses, dtype=np.float64))
    assert np.max(np.abs(curves[0] - curves[1]) / np.abs(curves[1])) <= 1e-4


def test_tiny_batch_trains_step_by_step_without_a_warning():
    solver = make_solver('lotka_volterra')
    eng = solver._get_engine()
    assert eng.info.small_batch_points == 0 and eng.lib.pinn_multi_step_max_points(eng.plan) == 0
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        solver.fit(niters=40, batch_size=50, lr=0.01)
    assert not [w for w in caught if 'pydens_b200' in str(w.message)]
    assert len(solver.losses) == 40 and np.isfinite(solver.losses[-1])


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpu_fit_matches_single_gpu(tmp_path):
    from test_gpu_multi import _run
    one = _run(1, str(tmp_path / 'w1.json'), problem='navier_stokes2d')
    two = _run(2, str(tmp_path / 'w2.json'), problem='navier_stokes2d')
    a, b = np.asarray(one['losses']), np.asarray(two['losses'])
    assert a.shape == b.shape == (30,) and two['allreduce'] == 'peer'
    assert np.max(np.abs(a - b) / np.abs(a)) <= 1e-4


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
def _create(spec, **kv):
    lib = N.load()
    plan = C.c_void_p()
    with env(**kv):
        rc = lib.pinn_plan_create(C.byref(spec), 0, C.byref(plan))
    if rc == 0:
        lib.pinn_plan_destroy(plan)
    return rc


def test_refusals():
    # a 64-wide network of 3 outputs with five channels: the thread kernel, never the tile kernels
    wide_cfg = dict(PC.PROBLEMS['navier_stokes2d'], features=[64, 64, 3])
    PC.PROBLEMS['_wide_ns'] = wide_cfg
    try:
        wspec = coupled_spec('_wide_ns')
        plan = Plan(wspec)
        assert plan.info.tensor_core == 0
        assert _create(wspec, PINN_FORCE_KERNEL='wide') == N.E_UNSUPPORTED
        assert _create(wspec, PINN_FORCE_KERNEL='wide128') == N.E_UNSUPPORTED
    finally:
        del PC.PROBLEMS['_wide_ns']
    lv = coupled_spec('lotka_volterra')                 # nf = 1, ns = 0: an order-3 plan of the same network
    lv.order = 3
    assert _create(lv) == N.E_UNSUPPORTED
    five = coupled_spec('navier_stokes2d')
    five.nf, five.ns = 5, 5
    assert _create(five) == N.E_UNSUPPORTED
    # through the Solver: the tracer refuses, backend='fused' raises, 'auto' trains on autograd with a warning
    kdv = lambda f, x, t: torch.cat([D(D(D(f[:, 0:1], x), x), x) + f[:, 1:2], D(f[:, 1:2], t)], dim=1)
    with pytest.raises(RuntimeError, match='fused'):
        Solver(kdv, ndims=2, layout='fafaf', features=[8, 8, 2], activation='Tanh', device='cuda', backend='fused')
    s = Solver(kdv, ndims=2, layout='fafaf', features=[8, 8, 2], activation='Tanh', device='cuda', backend='auto')
    with pytest.warns(UserWarning, match='autograd'):
        s.fit(niters=2, batch_size=64)
