""" The twelve-warp thread kernel (step_kernel_w12: 384 threads, three warps per scheduler) on the compact per-point
layout (build_remat_plan; its host-build twin is tests/test_occupancy_layout.py).  Plan creation places it for plain
one-output networks with two second-order directions whose compact storage fits twelve warps (cfg2: 147 rows per point,
168 registers, gradient accumulators in the workspace).  Checked against the fp64 oracle tensor by tensor at the bars of
test_gpu_placement.py, at batches of 1 and 33 points and one point either side of one and two full rounds of tiles, on
cfg2 and on networks at the forward / reverse block edges, with V in the equation and an initial condition; a step is
bit-reproducible, in-kernel sampling gives the bits of the same points passed in, and the in-kernel Adam tail follows
test_gpu_step_adam.py's per-element bars.  Residual layouts, oblique directions, variables in the initial condition and
networks whose compact storage does not fit twelve warps keep the placement and layout of before. """
import numpy as np
import pytest
import torch

import problems as P

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    import test_gpu_placement as TP
    import test_gpu_step_adam as TSA
    from helpers import rel_l2


def _poisson_v(f, x, y, D, V):
    return D(D(f, x), x) + D(D(f, y), y) - V('k', 1.5) * torch.sin(np.pi * (x + y))


def _wave_ic(f, x, t, D, V):
    return D(D(f, t), t) - 0.25 * D(D(f, x), x)


BASE = P.PROBLEMS['poisson2d']
CASES = {
    'cfg2': dict(BASE),
    'w1_1_1': dict(BASE, features=[1, 1, 1, 1], layout='fafafaf'),
    'w8_7_9': dict(BASE, features=[8, 7, 9, 1], layout='fafafaf'),
    'w16_9_15': dict(BASE, features=[16, 9, 15, 1], layout='fafafaf'),
    'w3_9_8_5': dict(BASE, features=[3, 9, 8, 5, 1], layout='fafafafaf'),
    'poisson_v': dict(BASE, equation=_poisson_v, features=[10, 12, 9, 1], layout='fafafaf', variables={'k': 1.5}),
    'wave_ic': dict(equation=_wave_ic, ndims=2, nparams=0, ic=P._ic_sin, bc=0, domain=(0, 1), features=[12, 10, 9, 1],
                    activation='Tanh', layout='fafafaf', ranges=[(0, 1), (0, 1)], log_scale=0.1),
}
# twelve warps of the compact layout do not fit shared memory: [16, 17, 15] needs 177 rows per point (148 fit)
TOO_WIDE = {'w16_17_15': dict(BASE, features=[16, 17, 15, 1], layout='fafafaf')}
OLD_LAYOUT = ['poisson_skip', 'mixed2d', 'heat1d_icvar'] + list(TOO_WIDE)


@pytest.fixture
def case(monkeypatch, request):
    name = request.param
    if name in CASES or name in TOO_WIDE:
        monkeypatch.setitem(P.PROBLEMS, name, {**CASES, **TOO_WIDE}[name])
    return name


def _engine(name, monkeypatch):
    solver, eng, (smem, warps, acc) = TP._placed_engine(name, 'default', monkeypatch)
    return solver, eng, smem, warps, acc


def _tensors(s, name):
    out = []
    for l in range(s.n_layers):
        out.append(('W%d' % l, slice(s.w_off[l], s.w_off[l] + s.widths[l] * s.widths[l + 1])))
        out.append(('b%d' % l, slice(s.b_off[l], s.b_off[l] + s.widths[l + 1])))
    end = s.b_off[s.n_layers - 1] + s.widths[s.n_layers]
    n_scalars = 1 + len(TP._cfg(name).get('variables') or {})
    return out + [('log_scale' if i == 0 else 'V%d' % i, slice(end + i, end + i + 1)) for i in range(n_scalars)]


@pytest.mark.parametrize('case', ['cfg2'], indirect=True)
def test_cfg2_runs_twelve_warps(case, monkeypatch):
    _, eng, smem, warps, acc = _engine(case, monkeypatch)
    info = eng.info
    assert (smem, warps, info.rows_per_point) == (True, 12, 147), (smem, warps, info.rows_per_point)
    assert info.regs_per_thread <= 168
    assert acc == 'per-warp, workspace'


@pytest.mark.parametrize('case', list(CASES), indirect=True)
def test_twelve_warps_match_fp64_oracle(case, monkeypatch):
    name = case
    solver, eng, smem, warps, acc = _engine(name, monkeypatch)
    assert (smem, warps) == (True, 12) and acc.startswith('per-warp'), (smem, warps, acc)
    params = solver.flat_params().cpu().numpy()
    round1 = 32 * warps * eng.info.sm_count
    sizes = [1, 33, round1 - 1, round1 + 1, 2 * round1 - 1, 2 * round1 + 1]
    pts, ref = TP._oracle_prefixes(name, params.astype(np.float64), sizes)
    tensors = _tensors(eng.spec, name)
    for n in sizes:
        loss, grads, residual = eng.loss_and_grads(pts[:n])
        grads, residual = grads.cpu().numpy(), residual.cpu().numpy()
        ref_loss, ref_res, ref_g, _ = ref[n]
        tag = '%s n=%d' % (name, n)
        cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(ref_res)))), 1e-30))
        assert np.isfinite(grads).all(), tag
        assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), tag
        assert rel_l2(residual, ref_res) <= 2e-5 * cond, tag
        assert rel_l2(grads[:ref_g.size], ref_g) <= 1e-4 * cond, tag
        scale = 1e-3 * np.linalg.norm(ref_g)
        for tname, sl in tensors:
            err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), scale, 1e-30)
            assert err <= 1e-4 * cond, '%s: %s rel err %.2e' % (tag, tname, err)
        # the same points again: the same bits
        loss2, grads2, residual2 = eng.loss_and_grads(pts[:n])
        assert loss2 == loss and np.array_equal(grads2.cpu().numpy(), grads) and np.array_equal(residual2.cpu().numpy(), residual), tag


@pytest.mark.parametrize('case', ['cfg2', 'w16_9_15'], indirect=True)
def test_twelve_warps_in_kernel_sampling_is_bit_reproducible(case, monkeypatch):
    _, eng, smem, warps, acc = _engine(case, monkeypatch)
    assert warps == 12
    n = 100000
    res = torch.empty(n, dtype=torch.float32, device=eng.device)
    eng._step(None, None, n, 1.0 / n, 0, residual=res, use_counter=False, step_value=3)
    runs = [(eng.out.clone(), res.clone())]
    pts = eng.sample(n, None, step=3)
    for _ in range(2):
        eng._step(pts, None, n, 1.0 / n, 0, residual=res, use_counter=False)
        runs.append((eng.out.clone(), res.clone()))
    torch.cuda.synchronize()
    assert torch.isfinite(runs[0][0]).all()
    for out, r in runs[1:]:
        assert torch.equal(out, runs[0][0]) and torch.equal(r, runs[0][1])


@pytest.mark.parametrize('case', ['cfg2', 'poisson_v'], indirect=True)
def test_twelve_warps_step_adam_per_element(case, monkeypatch):
    p, params, points, tag = TSA._thread(case, 'default', monkeypatch)
    assert '12 warps' in tag, tag
    rng = np.random.RandomState(5)
    TSA.adam_steps(tag, p, params, lambda s: TSA._device_points(points(TSA.N_ADAM, 300 + s)), rng, step0=37.0)


@pytest.mark.parametrize('case', OLD_LAYOUT, indirect=True)
def test_other_plans_keep_the_old_layout(case, monkeypatch):
    """ residual layouts, oblique directions, variables in the initial condition, and networks whose compact storage
    does not fit twelve warps: the placement of the eight-warp (or wider-jet) kernels, on the plan's own layout """
    _, eng, smem, warps, acc = _engine(case, monkeypatch)
    assert warps < 12 and eng.info.threads_per_cta != 384, (case, warps)
    if case in TOO_WIDE:
        assert eng.info.rows_per_point == 2 + 5 * (16 + 17 + 15 + 1) + eng.spec.n_slots
