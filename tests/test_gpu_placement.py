""" Every placement of the thread kernel (step_kernel / hi_step_kernel) against the fp64 oracle, and bit-reproducibility
under contention.  Plan creation places the kernel from its register count and the shared-memory budget: per-point
state in shared memory or in the per-warp global spill area, and the warp count per CTA.  Each warp accumulates its
gradient into an accumulator of its own (in shared memory, or in the workspace when that does not fit) and the CTA sums
them in warp order, so a step gives the same bits every time.  The placements are forced here through the overrides
plan creation reads (PINN_FORCE_MODE, PINN_GMEM_WARPS), and every test first checks from pinn_plan_info that the
placement it asked for is the one that runs.  PINN_FORCE_KERNEL=thread keeps the 64-wide networks off the tile kernel.

Batch sizes: 1 and 33; 32 * warps * sm_count +- 1, one point either side of the first full round of tiles (tiles are
dealt warp-slot-major); 200 003 (70 003 for the 64-wide networks, whose fp64 oracle costs ten times more CPU time, and
still above a full round of 16 warps on 132 SMs).  All sizes are prefixes of one batch, so the oracle runs once per problem over it and
its sums are cut at every prefix. """
import numpy as np
import pytest
import torch

import problems as P
import problems_systems as PS
from helpers import load_golden, rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from gpu_helpers import Replay
    from oracle import autograd_port as ap
    from pydens_b200 import Solver, D, V
    from test_gpu_systems import _check_against_golden


def _wave1d(f, x, t, D, V):
    return D(D(f, t), t) - D(D(f, x), x)


# 64-wide networks the tile kernel does not take (GELU, a residual layout): the thread kernel runs them by default,
# with about 110 KB of staged weights next to the per-warp accumulators
SYNTHETIC = {
    'gelu64': dict(equation=P._poisson2d, ndims=2, nparams=0, ic=None, bc=1, domain=(0, 1), features=[64, 64, 64, 1],
                   activation='GELU', layout='fafafaf', ranges=[(0, 1), (0, 1)]),
    'skip64': dict(equation=_wave1d, ndims=2, nparams=0, ic=P._ic_sin, bc=0, domain=(0, 1), features=[64, 64, 64, 1],
                   activation='Tanh', layout='fa R fa fa+ f', ranges=[(0, 1), (0, 1)], log_scale=0.1),
}
ORDER2 = [n for n in P.PROBLEMS if n not in P.HI_ORDER]
NAMES = ORDER2 + list(PS.PROBLEMS) + list(SYNTHETIC)
NO_SMEM_FORM = set(P.HI_DIRECTION) | set(P.HI_ORDER) | {'kdv_two_residuals'}    # global-memory state only

PLACEMENTS = {
    'default': {},
    'gmem': {'PINN_FORCE_MODE': 'gmem'},
    'smem': {'PINN_FORCE_MODE': 'smem'},
    'gmem_w1': {'PINN_FORCE_MODE': 'gmem', 'PINN_GMEM_WARPS': '1'},
    'gmem_w3': {'PINN_FORCE_MODE': 'gmem', 'PINN_GMEM_WARPS': '3'},
}
ORACLE_N = 200003


def _largest(name):
    return 70003 if max(_cfg(name)['features']) >= 64 else ORACLE_N


def _cfg(name):
    for reg in (P.PROBLEMS, PS.PROBLEMS, SYNTHETIC):
        if name in reg:
            return reg[name]
    raise KeyError(name)


def _ic(name, V_):
    cfg = _cfg(name)
    return cfg['ic_factory'](V_) if 'ic_factory' in cfg else cfg['ic']


def _solver(name):
    cfg = _cfg(name)
    torch.manual_seed(0)
    eq = cfg['equation']
    pkg_V = lambda n, init: V(n, data=torch.Tensor([init]))
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)           # systems: the [N, m] vs [N, 1] broadcast of the trial run
        solver = Solver(lambda u, *xs: eq(u, *xs, D=D, V=pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                        initial_condition=_ic(name, pkg_V), boundary_condition=cfg['bc'], domain=cfg['domain'],
                        layout=cfg['layout'], features=cfg['features'], activation=cfg['activation'],
                        device='cuda', backend='fused', seed=1234)
    if 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


def _oracle(name, params):
    cfg = _cfg(name)
    holder = {}
    ic = _ic(name, lambda n, init: holder['prob'].V(n, init))
    prob = ap.Problem(lambda u, *xs, D, V: cfg['equation'](u, *xs, D=D, V=V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                      initial_condition=ic, boundary_condition=cfg['bc'], domain=cfg['domain'], features=cfg['features'],
                      activation=cfg['activation'], dtype=torch.float64, variables=cfg.get('variables'),
                      layout=cfg['layout'])
    holder['prob'] = prob
    prob.load_flat(torch.as_tensor(params, dtype=torch.float64))
    return prob


def _points(name, n, seed):
    rng = np.random.RandomState(seed)
    return np.concatenate([rng.uniform(lo, hi, size=(n, 1)) for lo, hi in _cfg(name)['ranges']], axis=1).astype(np.float32)


# ---- the placement pinn_plan_info reports ------------------------------------------------------------------------------
def _align4(x):
    return (x + 3) & ~3


def _smem_bytes(eng, warps, n_wacc, state_in_smem):
    """ the step kernel's dynamic shared memory (pinn_step_kernel.cuh smem_layout) with `n_wacc` accumulators there """
    s = eng.spec
    wf = 0
    for l in range(s.n_layers):
        n_in, n_out = s.widths[l], s.widths[l + 1]
        p4, p8 = _align4(n_out), (n_in + 1 + 7) // 8 * 8
        wf += n_in * p4 + p4 * p8 + p4
    storage = max(eng.n_params, eng.info.rows_per_point * 32 * warps) if state_in_smem else eng.n_params
    return 4 * (_align4(wf) + _align4((eng.n_params + 4) * n_wacc) + 4 + _align4(storage))


def _placement(eng):
    """ -> (state in smem, warps per CTA, where the gradient accumulators are) """
    info = eng.info
    assert info.tensor_core == 0
    smem, warps = bool(info.activations_in_smem), info.threads_per_cta // 32
    acc = {_smem_bytes(eng, warps, 0, smem): 'per-warp, workspace',
           _smem_bytes(eng, warps, 1, smem): 'one per CTA, shared by all warps' if warps > 1 else 'per-warp, smem',
           _smem_bytes(eng, warps, warps, smem): 'per-warp, smem'}.get(info.smem_bytes, '?')
    return smem, warps, acc


def _placed_engine(name, placement, monkeypatch):
    monkeypatch.setenv('PINN_FORCE_KERNEL', 'thread')
    for k, v in PLACEMENTS[placement].items():
        monkeypatch.setenv(k, v)
    if placement == 'smem':
        if name in NO_SMEM_FORM:
            pytest.skip('this kernel keeps its per-point state in global memory only')
    solver = _solver(name)
    eng = solver._get_engine()
    if placement == 'smem' and _smem_bytes(eng, 1, 1, True) > torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 1024:
        pytest.skip('one warp of per-point state does not fit shared memory')
    smem, warps, acc = _placement(eng)
    want = {'gmem': (False, None), 'smem': (True, None), 'gmem_w1': (False, 1), 'gmem_w3': (False, 3)}.get(placement)
    if want is not None:
        assert smem == want[0], 'asked for %s, runs with state in %s' % (placement, 'smem' if smem else 'gmem')
        if want[1] is not None:
            assert warps == want[1], 'asked for %d warps, runs %d' % (want[1], warps)
    return solver, eng, (smem, warps, acc)


# ---- the fp64 oracle, once per problem ------------------------------------------------------------------------------
_ORACLE = {}


def _oracle_prefixes(name, params, cuts):
    """ fp64 oracle on prefixes of one batch: {n: (loss, residual [n], grads, u [n])}.  Computed segment by segment
    between the cuts (the loss and the gradients are means over the points: their sums add over segments). """
    key = (name, tuple(cuts))
    if key in _ORACLE:
        return _ORACLE[key]
    _ORACLE.clear()
    cfg = _cfg(name)
    pts = _points(name, max(cuts), seed=2024).astype(np.float64)
    prob = _oracle(name, params)
    bounds = sorted(set([0] + list(cuts)))
    sums, res, us = {}, [], []
    l_acc, g_acc = 0.0, None
    import warnings
    for a, b in zip(bounds[:-1], bounds[1:]):
        for c0 in range(a, b, 20000):
            c1 = min(b, c0 + 20000)
            with warnings.catch_warnings():
                warnings.simplefilter('ignore', UserWarning)
                l, r, g = prob.loss_and_grads(pts[c0:c1])
            l_acc += l * (c1 - c0)
            g = g.numpy() * (c1 - c0)
            g_acc = g if g_acc is None else g_acc + g
            res.append(PS.folded_residual(r, cfg['m']) if 'm' in cfg else r)
            us.append(prob.predict(pts[c0:c1]))
        sums[b] = (l_acc / b, np.concatenate(res), g_acc / b, np.concatenate(us))
    _ORACLE[key] = (pts.astype(np.float32), sums)
    return _ORACLE[key]


def _cuts(name, sm_count):
    return sorted({1, 33, _largest(name)} | {32 * w * sm_count + d for w in range(1, 17) for d in (-1, 1)
                                             if 32 * w * sm_count + d < _largest(name)})


@pytest.mark.parametrize('placement', list(PLACEMENTS))
@pytest.mark.parametrize('name', NAMES)
def test_placement_matches_fp64_oracle(name, placement, monkeypatch):
    solver, eng, (smem, warps, acc) = _placed_engine(name, placement, monkeypatch)
    assert acc.startswith('per-warp'), '%s: gradient accumulators %s' % (placement, acc)
    params = solver.flat_params().cpu().numpy()
    pts, ref = _oracle_prefixes(name, params.astype(np.float64), _cuts(name, eng.info.sm_count))
    s = eng.spec
    tensors = []
    for l in range(s.n_layers):
        tensors.append(('W%d' % l, slice(s.w_off[l], s.w_off[l] + s.widths[l] * s.widths[l + 1])))
        tensors.append(('b%d' % l, slice(s.b_off[l], s.b_off[l] + s.widths[l + 1])))
    end = s.b_off[s.n_layers - 1] + s.widths[s.n_layers]
    n_scalars = 1 + len(_cfg(name).get('variables') or {})                 # log_scale, then the equation variables
    tensors += [('log_scale' if i == 0 else 'V%d' % i, slice(end + i, end + i + 1)) for i in range(n_scalars)]
    round1 = 32 * warps * eng.info.sm_count
    for n in (1, 33, round1 - 1, round1 + 1, _largest(name)):
        loss, grads, residual = eng.loss_and_grads(pts[:n])
        grads, residual = grads.cpu().numpy(), residual.cpu().numpy()
        ref_loss, ref_res, ref_g, ref_u = ref[n]
        tag = '%s %s (%s, %d warps, %s) n=%d' % (name, placement, 'smem' if smem else 'gmem', warps, acc, n)
        # tolerances and cancellation factor of test_gpu_fuzz.py
        cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(ref_res)))), 1e-30))
        assert np.isfinite(grads).all(), tag
        assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), tag
        assert rel_l2(residual, ref_res) <= 2e-5 * cond, tag
        assert rel_l2(grads[:ref_g.size], ref_g) <= 1e-4 * cond, tag
        scale = 1e-3 * np.linalg.norm(ref_g)           # a tensor whose gradient is 1000x below the whole is held to that
        for tname, sl in tensors:
            err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), scale, 1e-30)
            assert err <= 1e-4 * cond, '%s: %s rel err %.2e' % (tag, tname, err)
        u = solver.predict(*[pts[:n, i] for i in range(pts.shape[1])]).reshape(-1)
        assert np.abs(u - ref_u).max() <= 1e-5 * max(1.0, np.abs(ref_u).max()), tag


@pytest.mark.parametrize('placement', list(PLACEMENTS))
@pytest.mark.parametrize('name', [n for n in NAMES if n not in SYNTHETIC])
def test_golden_points_under_every_placement(name, placement, monkeypatch):
    g = load_golden(name)
    solver, eng, _ = _placed_engine(name, placement, monkeypatch)
    solver.load_flat_params(g['params'])
    loss, grads, residual = eng.loss_and_grads(g['points'])
    grads, residual = grads.cpu().numpy(), residual.cpu().numpy()
    u = solver.predict(*[g['points'][:, i] for i in range(g['points'].shape[1])]).reshape(-1)
    if name in PS.PROBLEMS:
        _check_against_golden(name, g, loss, residual, grads, u, eng.spec)
        return
    assert abs(loss - float(g['loss'])) <= 1e-5 * abs(float(g['loss']))
    assert rel_l2(residual, g['residual']) <= 1e-5
    assert rel_l2(grads, g['grads']) <= 1e-4
    s = eng.spec
    for l in range(s.n_layers):
        w = slice(s.w_off[l], s.w_off[l] + s.widths[l] * s.widths[l + 1])
        b = slice(s.b_off[l], s.b_off[l] + s.widths[l + 1])
        assert rel_l2(grads[w], g['grads'][w]) <= 1e-4, 'W%d' % l
        assert rel_l2(grads[b], g['grads'][b]) <= 1e-4, 'b%d' % l
    assert rel_l2(u, g['u']) <= 1e-5


# ---- bit-reproducibility under contention ---------------------------------------------------------------------------
# ode_param at its BASELINE size (cfg3) and ode_var: 15-16 warps share a CTA; wave3d and the 64-wide networks: global
# state, eight warps, with the staged weights taking most of shared memory; every forced placement of the step kernel;
# the five / six-direction and whole-jet kernels
REPRO = ([('ode_param', 'default'), ('ode_var', 'default'), ('wave3d', 'default'), ('gelu64', 'default'),
          ('skip64', 'default'), ('hess3d', 'default'), ('heat4d', 'default'), ('kdv', 'default'), ('beam', 'default')]
         + [('ode_param', p) for p in PLACEMENTS if p != 'default'] + [('gelu64', p) for p in ('gmem_w1', 'gmem_w3')])


@pytest.mark.parametrize('name,placement', REPRO)
def test_step_is_bit_reproducible(name, placement, monkeypatch):
    solver, eng, (smem, warps, acc) = _placed_engine(name, placement, monkeypatch)
    n = 1000000
    tag = '%s %s (%s, %d warps, accumulators %s)' % (name, placement, 'smem' if smem else 'gmem', warps, acc)
    res = torch.empty(n, dtype=torch.float32, device=eng.device)
    eng._step(None, None, n, 1.0 / n, 0, residual=res, use_counter=False, step_value=3)
    runs = [(eng.out.clone(), res.clone())]
    pts = eng.sample(n, None, step=3)
    for _ in range(3):
        eng._step(pts, None, n, 1.0 / n, 0, residual=res, use_counter=False)
        runs.append((eng.out.clone(), res.clone()))
    torch.cuda.synchronize()
    assert torch.isfinite(runs[0][0]).all(), tag
    for i, (out, r) in enumerate(runs[1:]):
        nd = int((out != runs[0][0]).sum())
        assert torch.equal(out, runs[0][0]), '%s: run %d differs from the in-kernel-sampled step in %d of %d outputs' % (
            tag, i + 1, nd, out.numel())
        assert torch.equal(r, runs[0][1]), '%s: residual of run %d differs' % (tag, i + 1)
    assert acc.startswith('per-warp'), tag


def test_persistent_multi_step_kernel_is_bit_reproducible(monkeypatch):
    """ multi_step_kernel (one CTA, every warp busy) on a fixed batch: two fits from the same state end on the same bits """
    monkeypatch.setenv('PINN_MULTI_KERNEL', 'tile')
    monkeypatch.setenv('PINN_FORCE_KERNEL', 'thread')
    import warnings
    eng = _solver('ode_param')._get_engine()
    n = min(8192, int(eng.lib.pinn_multi_step_max_points(eng.plan)))
    assert n >= 1024
    batches = [P.make_points('ode_param', n, seed=50 + i) for i in range(6)]
    finals = []
    for _ in range(2):
        solver = _solver('ode_param')
        with warnings.catch_warnings():
            warnings.simplefilter('error', UserWarning)        # "steps_per_launch ignored" must not happen
            solver.fit(niters=6, batch_size=n, sampler=Replay(list(batches)), lr=0.01, steps_per_launch=6)
        finals.append((solver.flat_params().cpu(), np.asarray(solver.losses)))
    assert torch.equal(finals[0][0], finals[1][0])
    assert np.array_equal(finals[0][1], finals[1][1])
