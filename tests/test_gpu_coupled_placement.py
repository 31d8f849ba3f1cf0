""" The coupled-system thread kernel (coupled_step_kernel<NF, NS, GMEM, MAXT> with coupled_forward_kernel<GMEM>) at
every placement, width edge and batch edge against the fp64 oracle, through the bare C ABI (pinn_step + pinn_forward).
CPU twin of the width cases: test_coupled_widths.py.

- placement: the five placements of test_gpu_placement.py under PINN_FORCE_KERNEL=thread on Navier-Stokes-like k = 3
  networks from 20 to 128 units wide, a 48-64-wide k = 2 network with GELU and one with a residual layout (the tile
  classes refuse both), and a k = 4 residual SiLU network.  Each case first checks from pinn_plan_info that the
  placement it asked for runs (state in smem or gmem, warps, and where the per-warp gradient accumulators live), then
  steps batch prefixes 1, 33, 32 * warps * sm_count +- 1 and 200 003 (70 003 for networks 64 or more wide).  The
  matrix reaches state in smem and gmem, each with the accumulators in smem and in the workspace, and both forms of
  the forward kernel;
- width edges: the cases of test_coupled_widths.py (every jet set at widths 1..64, (2, 2) and (4, 4) at every block
  edge up to 128, uneven layers, V in the equation and the initial condition, 6..8 columns), default placement and,
  for widths of 64 and up, one warp with state in global memory;
- the widest two-layer network the thread kernel plans for k = 2, 3, 4, found by plan creation, and what takes one
  unit more;
- the thread kernel against the coupled 128-wide tile kernel on the networks both hold;
- bit-reproducibility at the workspace-accumulator placements and in-kernel sampling on a wide network;
- the in-kernel Adam fit at the workspace placement against the fp64 port's own fit;
- L1 / Huber / SmoothL1 / MSE-sum on a wide network with the accumulators in the workspace.
Bars: those of test_gpu_coupled.py (loss and residual 2e-5 cond, gradients 1e-4 cond whole and 2e-4 cond per tensor,
u 1e-5). """
import contextlib
import types
import warnings

import numpy as np
import pytest
import torch

import problems_coupled as PC
from helpers import rel_l2
from test_coupled_widths import CASES, _seed_where
from test_gpu_placement import PLACEMENTS, _placement, _smem_bytes

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(2400)]

if torch.cuda.is_available():
    from gpu_helpers import Replay
    from oracle import autograd_port as ap
    from pydens_b200 import _native as N
    from test_coupled import coupled_oracle, folded, oracle_loss_and_grads, random_setup, tolerances
    from test_gpu_coupled import Plan, check_tensors, env, make_solver
    from test_gpu_tile128_coupled import Case, _create_rc

WIDE = [[128, 128], [100, 72], [65, 16], [128, 16, 128]]          # 65-128 wide: the thread kernel holds them


def _networks():
    """ name -> (seed, random_coupled overrides) of the placement matrix """
    nets = {'ns_20x2': (11, dict(k=3, jet=(2, 2), hidden=[20, 20])),
            'ns_64x3': (12, dict(k=3, jet=(2, 2), hidden=[64, 64, 64]))}
    for i, h in enumerate(WIDE):
        nets['ns_' + 'x'.join(map(str, h))] = (13 + i, dict(k=3, jet=(2, 2), hidden=h))
    nets['gelu_48x64_k2'] = (_seed_where(100, lambda c: 'GELU' in c['acts'], k=2, jet=(2, 1), hidden=[48, 64]),
                             dict(k=2, jet=(2, 1), hidden=[48, 64]))
    nets['resnet_56_k2'] = (_seed_where(200, lambda c: c['layout'].startswith('faR'), k=2, jet=(2, 2), hidden=56),
                            dict(k=2, jet=(2, 2), hidden=56))
    nets['resnet_silu_40_k4'] = (_seed_where(300, lambda c: c['layout'].startswith('faR') and 'SiLU' in c['acts'],
                                             k=4, jet=(3, 3), hidden=40), dict(k=4, jet=(3, 3), hidden=40))
    return nets


NETS = _networks()
ORACLE_N = 200003


def _largest(features):
    return 70003 if max(features[:-1]) >= 64 else ORACLE_N


def _setup(net, n=1):
    seed, fixed = NETS[net]
    return random_setup(seed, kind='mse', n=n, **fixed)


# ---- placement ----------------------------------------------------------------------------------------------------------
def _plan(spec, placement):
    with env(PINN_FORCE_KERNEL='thread', **PLACEMENTS[placement]):
        return Plan(spec)


def _fwd_in_gmem(spec, info):
    """ the forward kernel's placement (pinn_kernels.cu place_forward_kernel): eight warps of fwd_rows rows each """
    units = sum(spec.widths[l + 1] for l in range(spec.n_layers))
    units += sum(spec.widths[l + 1] for l in range(spec.n_layers) if spec.skip_src[l] >= 0)
    fwd_rows = spec.widths[0] + units + spec.n_slots
    wf = 0
    for l in range(spec.n_layers):
        n_in, n_out = spec.widths[l], spec.widths[l + 1]
        p4, p8 = (n_out + 3) // 4 * 4, (n_in + 1 + 7) // 8 * 8
        wf += n_in * p4 + p4 * p8 + p4
    total = (wf + 3) // 4 * 4 + 4 + (max(spec.n_params, fwd_rows * 32 * 8) + 3) // 4 * 4
    return total * 4 > torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 64, fwd_rows


def _ws_bytes(plan, smem, warps, acc_ws, fwd_gmem, fwd_rows):
    """ pinn_workspace_bytes as the placement implies it: ticket, partials, per-warp accumulators, the larger spill """
    s, sm = plan.spec, plan.info.sm_count
    up = lambda b: (b + 255) & ~255
    off = up(256 + sm * (s.n_params + 4) * 4)
    off = up(off + (sm * warps * (s.n_params + 4) * 4 if acc_ws else 0))
    spill = 0 if smem else sm * warps * plan.info.rows_per_point * 32 * 4
    return off + max(spill, sm * 8 * fwd_rows * 32 * 4 if fwd_gmem else 0)


def placed(spec, placement):
    """ -> (plan, (state in smem, warps, accumulators, forward state in gmem)); skips where a forced placement
    cannot fit, and fails where the plan runs another placement than the one asked for """
    plan = _plan(spec, placement)
    eng = types.SimpleNamespace(info=plan.info, spec=spec, n_params=spec.n_params)
    assert plan.info.tensor_core == 0 and plan.info.small_batch_points == 0
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    if placement == 'smem' and not plan.info.activations_in_smem and _smem_bytes(eng, 1, 1, True) > optin - 1024:
        pytest.skip('one warp of per-point state does not fit shared memory')
    smem, warps, acc = _placement(eng)
    assert acc.startswith('per-warp'), '%s: gradient accumulators %s' % (placement, acc)
    want = {'gmem': (False, None), 'smem': (True, None), 'gmem_w1': (False, 1), 'gmem_w3': (False, 3)}.get(placement)
    if want is not None:
        assert smem == want[0], 'asked for %s, runs with state in %s' % (placement, 'smem' if smem else 'gmem')
        assert want[1] is None or warps == want[1], 'asked for %d warps, runs %d' % (want[1], warps)
    fwd_gmem, fwd_rows = _fwd_in_gmem(spec, plan.info)
    ws = plan.lib.pinn_workspace_bytes(plan.plan, 1)
    assert ws == _ws_bytes(plan, smem, warps, acc == 'per-warp, workspace', fwd_gmem, fwd_rows), ws
    return plan, (smem, warps, 'workspace' if acc == 'per-warp, workspace' else 'smem', fwd_gmem)


def _points(cfg, n, seed=2024):
    """ n points of the problem's domain (and [0, 1] parameter columns), 1e-3 of the width away from the faces """
    rng = np.random.RandomState(seed)
    ranges = list(cfg['domain']) + [(0.0, 1.0)] * cfg['nparams']
    return np.concatenate([rng.uniform(lo + 1e-3 * (hi - lo), hi - 1e-3 * (hi - lo), size=(n, 1)) for lo, hi in ranges],
                          axis=1).astype(np.float32)


_ORACLE = {}


def _oracle_prefixes(net, sm_count):
    """ (cfg, params, spec, points, {n: (loss, residual [n, k], grads, u [n, k])}) of one batch, its prefixes cut at 1,
    33, every 32 * warps * sm_count +- 1 and the largest size; segment sums (loss and gradients are means) """
    if net not in _ORACLE:
        cfg, prob, params, _, _, spec = _setup(net)
        big = _largest(cfg['features'])
        cuts = sorted({1, 33, big} | {32 * w * sm_count + d for w in range(1, 17) for d in (-1, 1)
                                      if 32 * w * sm_count + d < big})
        pts = _points(cfg, big)
        bounds = sorted(set([0] + cuts + list(range(0, big, 20000))))
        ref, res, us, l_acc, g_acc = {}, [], [], 0.0, 0.0
        for a, b in zip(bounds[:-1], bounds[1:]):
            l, r, g = oracle_loss_and_grads(prob, pts[a:b].astype(np.float64))
            l_acc, g_acc = l_acc + l * (b - a), g_acc + g.numpy() * (b - a)
            res.append(np.asarray(r).reshape(b - a, -1))
            us.append(prob.predict(pts[a:b].astype(np.float64)).reshape(b - a, -1))
            if b in cuts:
                ref[b] = (l_acc / b, np.concatenate(res), g_acc / b, np.concatenate(us))
        _ORACLE.clear()
        _ORACLE[net] = (cfg, params, spec, pts, ref)
    return _ORACLE[net]


def check_step(tag, spec, k, got, ref):
    """ loss, folded residual, every tensor and u [n, k] against the fp64 oracle at the bars of test_gpu_coupled.py;
    -> the relative errors """
    loss, residual, grads, u = got
    ref_loss, ref_res, ref_g, ref_u = ref
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(ref_res)))), 1e-30))
    err = dict(loss=abs(loss - ref_loss) / max(abs(ref_loss), 1e-6), res=rel_l2(residual, folded(ref_res, k)),
               grads=rel_l2(grads, ref_g), u=rel_l2(u, ref_u))
    assert np.isfinite(grads).all(), tag
    assert err['loss'] <= 2e-5 * cond, '%s %s' % (tag, err)
    assert err['res'] <= 2e-5 * cond, '%s %s' % (tag, err)
    assert err['grads'] <= 1e-4 * cond, '%s %s' % (tag, err)
    check_tensors(spec, grads, ref_g, 2e-4 * cond)
    assert u.shape == ref_u.shape and err['u'] <= 1e-5, '%s %s' % (tag, err)
    return err


@pytest.mark.parametrize('placement', list(PLACEMENTS))
@pytest.mark.parametrize('net', list(NETS))
def test_placement_matches_fp64_oracle(net, placement):
    cfg0, _, _, _, _, spec = _setup(net)
    plan, (smem, warps, acc, fwd_gmem) = placed(spec, placement)
    cfg, params, spec, pts, ref = _oracle_prefixes(net, plan.info.sm_count)
    tag = '%s %s (state %s, %d warps, accumulators %s, forward state %s)' % (
        net, placement, 'smem' if smem else 'gmem', warps, acc, 'gmem' if fwd_gmem else 'smem')
    worst = {}
    round1 = 32 * warps * plan.info.sm_count
    for n in (1, 33, round1 - 1, round1 + 1, _largest(cfg['features'])):
        err = check_step('%s n=%d' % (tag, n), spec, cfg['k'], plan.step(params, pts[:n]), ref[n])
        worst = {key: max(v, worst.get(key, 0.0)) for key, v in err.items()}
    print('%s: worst rel err %s' % (tag, ', '.join('%s %.2e' % kv for kv in worst.items())))


def test_matrix_reaches_every_state_and_accumulator_placement():
    """ state in smem / gmem x accumulators in smem / the workspace, all with k > 1; and the forward kernel's
    global-memory form """
    seen, fwd = set(), set()
    for net in NETS:
        spec = _setup(net)[-1]
        for placement in PLACEMENTS:
            plan = _plan(spec, placement)
            eng = types.SimpleNamespace(info=plan.info, spec=spec, n_params=spec.n_params)
            smem, _, acc = _placement(eng)
            seen.add((smem, acc == 'per-warp, workspace'))
            fwd.add(_fwd_in_gmem(spec, plan.info)[0])
    assert seen == {(True, False), (True, True), (False, False), (False, True)}, seen
    assert fwd == {True, False}


# ---- width edges ----------------------------------------------------------------------------------------------------------
WIDTH_N = 3001


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_width_edge_matches_fp64_oracle(case):
    _, seed, fixed = case
    cfg, prob, params, pts, (_, _, _, r64, thr), spec = random_setup(seed, kind='mse', n=WIDTH_N, **fixed)
    l, r, g = oracle_loss_and_grads(prob, pts.astype(np.float64))
    ref = (l, np.asarray(r), g.numpy(), prob.predict(pts.astype(np.float64)).reshape(-1, cfg['k']))
    placements = ['default'] + (['gmem_w1'] if max(cfg['features'][:-1]) >= 64 else [])
    for placement in placements:
        with env(**PLACEMENTS[placement]):
            plan = Plan(spec)
        assert plan.info.tensor_core == 0
        if placement == 'gmem_w1':
            assert not plan.info.activations_in_smem and plan.info.threads_per_cta == 32
        check_step('%s %s %s' % (cfg['tag'], cfg['features'], placement), spec, cfg['k'], plan.step(params, pts), ref)


# ---- the widest networks the thread kernel plans ----------------------------------------------------------------------------
def _two_layer(k, w, n=1):
    return Case(40 + k, [(w, 'Tanh'), (w, 'Tanh')], n=n, k=k, jet=(2, 2), kind='mse')


@pytest.mark.parametrize('k', [2, 3, 4])
def test_widest_network_the_thread_kernel_plans(k):
    lo, hi = 1, 512                                # lo plans, hi does not
    assert _create_rc(_two_layer(k, lo).spec, 'thread')[0] == 0
    assert _create_rc(_two_layer(k, hi).spec, 'thread')[0] == N.E_UNSUPPORTED
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _create_rc(_two_layer(k, mid).spec, 'thread')[0] == 0:
            lo = mid
        else:
            hi = mid
    case = _two_layer(k, lo, n=20011)
    print('k=%d: the thread kernel plans up to two %d-wide layers' % (k, lo))
    plan = _plan(case.spec, 'default')
    loss, residual, grads, u = plan.step(case.params, case.pts)
    l, r, g = case.oracle()
    check_step('k=%d w=%d' % (k, lo), case.spec, k, (loss, residual, grads, u),
               (l, r, g, case.prob.predict(case.pts.astype(np.float64)).reshape(-1, k)))
    wider = _two_layer(k, lo + 1).spec
    assert _create_rc(wider, 'thread')[0] == N.E_UNSUPPORTED
    rc, info = _create_rc(wider, None)
    if lo + 1 <= 128:
        assert rc == 0 and info.tensor_core == 2, (lo + 1, rc)
    else:
        assert rc == N.E_UNSUPPORTED, (lo + 1, rc)


# ---- the thread kernel against the 128-wide tile kernel --------------------------------------------------------------------
@pytest.mark.parametrize('hidden', WIDE[:3], ids=['x'.join(map(str, h)) for h in WIDE[:3]])
def test_thread_kernel_agrees_with_the_128_wide_class(hidden):
    """ independent of the oracle: two fp32 kernels with different summation orders on the same 50 001 points.  Each
    is within 1e-4 cond of the fp64 oracle; between them the difference is the rounding of the fp32 sums over 50 001
    points and 128 inputs: on an H100 80GB HBM3 the gradients differ by 4.9e-7 to 7.8e-7 relative L2, the loss by at
    most 1.7e-7 and u not at all (DESIGN section 8: 7.8e-7 for the one-output pair), so 2e-5 leaves a factor 25 """
    case = Case(7, [(w, 'Tanh') for w in hidden], n=50001, k=3, jet=(2, 2), kind='mse')
    thread = Plan(case.spec)
    assert thread.info.tensor_core == 0
    with env(PINN_FORCE_KERNEL='wide128'):
        tile = Plan(case.spec)
    assert tile.info.tensor_core == 2
    a, b = thread.step(case.params, case.pts), tile.step(case.params, case.pts)
    err = dict(loss=abs(a[0] - b[0]) / abs(b[0]), res=rel_l2(a[1], b[1]), grads=rel_l2(a[2], b[2]), u=rel_l2(a[3], b[3]))
    print('%s thread vs 128-wide tile: %s' % (hidden, ', '.join('%s %.2e' % kv for kv in err.items())))
    assert err['loss'] <= 1e-5 and err['res'] <= 1e-5 and err['grads'] <= 2e-5 and err['u'] <= 1e-5, err
    check_tensors(case.spec, a[2], b[2], 4e-5)


# ---- bit level ------------------------------------------------------------------------------------------------------------
REPRO = [(net, p) for net in ('ns_128x128', 'ns_100x72', 'gelu_48x64_k2') for p in PLACEMENTS] + [('ns_128x16x128', 'gmem_w3')]


@pytest.mark.parametrize('net,placement', REPRO)
def test_step_is_bit_reproducible(net, placement):
    cfg, _, params, _, _, spec = _setup(net)
    pts = _points(cfg, 300007, seed=7)
    plan, (smem, warps, acc, _) = placed(spec, placement)
    if acc != 'workspace' and placement != 'gmem_w3':
        pytest.skip('accumulators in shared memory at this placement: not one of the cases of this test')
    runs = [plan.step(params, pts) for _ in range(2)]
    tag = '%s %s (%s, %d warps, accumulators %s)' % (net, placement, 'smem' if smem else 'gmem', warps, acc)
    assert np.isfinite(runs[0][2]).all(), tag
    for x, y in zip(runs[0], runs[1]):
        assert np.array_equal(np.asarray(x), np.asarray(y)), tag


@contextlib.contextmanager
def _wide_ns():
    """ the Navier-Stokes problem of problems_coupled.py on [2, 100, 100, 3] (per-warp accumulators in the workspace) """
    PC.PROBLEMS['_ns_100x100'] = dict(PC.PROBLEMS['navier_stokes2d'], features=[100, 100, 3])
    try:
        yield '_ns_100x100'
    finally:
        del PC.PROBLEMS['_ns_100x100']


def _wide_ns_solver():
    with _wide_ns() as name:
        return make_solver(name)


def test_in_kernel_sampling_equals_explicit_points_on_a_wide_network():
    eng = _wide_ns_solver()._get_engine()
    assert eng.info.tensor_core == 0
    n = 70001
    outs = []
    for _ in range(2):
        eng._step(None, None, n, 1.0 / n, 0, use_counter=False, step_value=5)
        torch.cuda.synchronize()
        outs.append(eng.out.clone())
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
    pts = eng.sample(n, step=5)
    eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
    torch.cuda.synchronize()
    assert torch.equal(eng.out, outs[0]), int((eng.out != outs[0]).sum())


# ---- the in-kernel Adam fit at the workspace placement --------------------------------------------------------------------
@pytest.mark.parametrize('fused_adam', ['1', '0'])
def test_fit_follows_the_fp64_port_fit(fused_adam):
    """ Solver.fit on Navier-Stokes [2, 100, 100, 3] (accumulators in the workspace) against oracle.autograd_port.fit
    in fp64 from the same weights on the same batches; bars of test_gpu_coupled.test_fit_follows_the_reference_fit """
    niters, batch, lr = 15, 4096, 0.002
    solver = _wide_ns_solver()
    eng = solver._get_engine()
    assert _placement(eng)[2] == 'per-warp, workspace'
    params = solver.flat_params().cpu().numpy().copy()
    batches = [PC.make_points('navier_stokes2d', batch, seed=3000 + i) for i in range(niters)]
    with env(PYDENS_B200_FUSED_ADAM=fused_adam), warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        solver.fit(niters=niters, batch_size=batch, sampler=Replay(list(batches)), lr=lr)
    assert not [w for w in caught if 'pydens_b200' in str(w.message)]
    with _wide_ns() as name:
        prob = coupled_oracle(name, params=params[:eng.n_params].astype(np.float64))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        ref = np.asarray(ap.fit(prob, niters, batch, lr=lr, point_stream=lambda i: torch.as_tensor(batches[i], dtype=torch.float64)),
                         dtype=np.float64)
    losses = np.asarray(solver.losses, dtype=np.float64)
    assert losses.shape == ref.shape
    assert np.max(np.abs(losses - ref) / np.abs(ref)) <= 2e-3, (losses, ref)
    flat = solver.flat_params().cpu().numpy()[:eng.n_params]
    assert rel_l2(flat, prob.flat_params().numpy()) <= 1e-3


# ---- criteria on a wide network ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['l1', 'huber', 'smooth_l1', 'mse_sum'])
def test_criteria_on_a_wide_network_match_torch_on_the_fp64_oracle(kind):
    cfg, prob, params, pts, (key, crit, red, r64, thr), spec = random_setup(21, k=3, jet=(2, 2), kind=kind,
                                                                             hidden=[100, 100], n=20011)
    plan, (smem, warps, acc, _) = placed(spec, 'default')
    assert acc == 'workspace', acc
    loss, residual, grads, _ = plan.step(params, pts)
    weight = float(cfg['n']) if red == 'sum' else 1.0
    ref_loss, ref_res, ref_grads = oracle_loss_and_grads(prob, pts.astype(np.float64), criterion=crit)
    cond, slack = tolerances(cfg, r64, thr)
    grads = grads * np.float32(weight)
    assert abs(loss * weight - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), cfg['tag']
    assert rel_l2(grads, ref_grads.numpy()) <= 1e-4 * cond * slack, cfg['tag']
    check_tensors(spec, grads, ref_grads.numpy(), 2e-4 * cond * slack)
    if kind == 'mse_sum':
        assert rel_l2(residual, folded(ref_res, 3, key)) <= 2e-5 * cond, cfg['tag']
