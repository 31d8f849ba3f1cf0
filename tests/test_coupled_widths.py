""" Coupled systems (networks with 2..4 outputs) at the width edges of the thread kernel's reverse sweep, on the host
build of the device code (tests/emul, point_step / point_forward with MULTI) against the fp64 oracle.  The GPU twin,
test_gpu_coupled_placement.py, runs the same cases on coupled_step_kernel / coupled_forward_kernel; this file keeps
the math the two share checked on every CPU run.

bwd_layer reduces a layer's weight gradient in blocks of 8 input columns plus the bias column (n_in + 1 padded to a
multiple of 8): a hidden width that is a multiple of 8 puts the bias into a block of its own, and the output layer
(k rows of a 4-row block, the rows past k masked) takes the last hidden width as its n_in.  A hidden width of 1 runs
the one-unit form as a hidden layer under the k-output layer.  The cases:
- every jet set at hidden widths 1, 8, 16, 33 and 64, k rotating over 2, 3 and 4 (residual layouts where drawn);
- (nf, ns) = (2, 2) and (4, 4) at every width from 1 to 128 that sits on or next to a block edge;
- uneven hidden layers, so that the output layer's n_in and the hidden widths sit on different edges;
- V in the equation and in the initial condition, and 6..8 point columns (parameters as extra columns).
Bars: those of test_coupled.py's random problems (loss 2e-5 cond, gradient 1e-4 cond, residual 2e-5 cond, u 1e-5),
and every tensor to 2e-4 cond (test_gpu_coupled.check_tensors). """
import numpy as np
import pytest

import emul_coupled as EC
from helpers import rel_l2
from test_coupled import JET_SETS, folded, oracle_loss_and_grads, random_coupled, random_setup, tolerances
from test_gpu_coupled import check_tensors

EDGE_WIDTHS = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 24, 31, 32, 33, 48, 63, 64, 65, 100, 128]
UNEVEN = [[33, 8], [8, 33], [1, 16], [16, 1], [65, 17], [17, 65], [128, 1], [1, 128], [24, 1, 33], [9, 64, 7]]
N_POINTS = 37                       # a warp tile and a few points of the next


def _seed_where(start, pred, **fixed):
    """ the first seed from `start` whose drawn problem satisfies `pred` (fixed draws: see random_coupled) """
    for seed in range(start, start + 1000):
        if pred(random_coupled(seed, **fixed)):
            return seed
    raise ValueError('no seed in %d..%d draws such a problem' % (start, start + 999))


def _both_vars(cfg):
    return set(cfg['variables']) == {'a', 'c'}


def width_cases():
    """ (id, seed, random_coupled overrides): the width, jet set and column cases of this file and its GPU twin """
    cases = []
    for i, jet in enumerate(JET_SETS):
        for w_i, w in enumerate([1, 8, 16, 33, 64]):
            k = 2 + (5 * i + w_i) % 3
            cases.append(('nf%d_ns%d_w%d_k%d' % (jet + (w, k)), 5000 + 17 * i + w_i, dict(k=k, jet=jet, hidden=w)))
    for jet in [(2, 2), (4, 4)]:
        for w_i, w in enumerate(EDGE_WIDTHS):
            k = 2 + w_i % 3
            cases.append(('edge_nf%d_ns%d_w%d_k%d' % (jet + (w, k)), 6000 + 100 * jet[0] + w_i, dict(k=k, jet=jet, hidden=w)))
    for u_i, hidden in enumerate(UNEVEN):
        jet, k = [(2, 2), (4, 4), (2, 1), (1, 0), (3, 3)][u_i % 5], 2 + u_i % 3
        cases.append(('nf%d_ns%d_w%s_k%d' % (jet + ('x'.join(map(str, hidden)), k)), 7000 + u_i,
                      dict(k=k, jet=jet, hidden=hidden)))
    # V in the equation and in the initial condition (its partials for every component), at the block edges
    for v_i, (jet, hidden) in enumerate([((2, 2), 16), ((2, 1), 33), ((2, 0), [8, 17]), ((3, 3), 64), ((2, 2), [1, 24])]):
        k = 2 + v_i % 3
        seed = _seed_where(8000 + 50 * v_i, _both_vars, k=k, jet=jet)
        cases.append(('vars_nf%d_ns%d_k%d_%d' % (jet + (k, v_i)), seed, dict(k=k, jet=jet, hidden=hidden)))
    # 6..8 point columns: parameters the network takes as inputs
    for c_i, (jet, cols, hidden) in enumerate([((1, 1), 8, 16), ((2, 2), 7, 33), ((3, 2), 6, [8, 64]), ((4, 4), 8, 17)]):
        k = 2 + c_i % 3
        seed = 9000 + c_i
        ndims = random_coupled(seed, k=k, jet=jet)['ndims']
        cases.append(('cols%d_nf%d_ns%d_k%d' % ((cols,) + jet + (k,)), seed,
                      dict(k=k, jet=jet, hidden=hidden, nparams=cols - ndims)))
    return cases


CASES = width_cases()


def check_against_oracle(cfg, prob, spec, pts, got, u, r64, thr):
    """ loss, folded residual, the whole gradient, every tensor and u [n, k] against the fp64 oracle (MSE) """
    loss, residual, grads = got
    ref_loss, ref_res, ref_grads = oracle_loss_and_grads(prob, pts.astype(np.float64))
    ref_grads = ref_grads.numpy()
    cond, _ = tolerances(cfg, r64, thr)
    k, tag = cfg['k'], '%s %s' % (cfg['tag'], cfg['features'])
    assert np.isfinite(grads).all(), tag
    assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), tag
    assert rel_l2(residual, folded(ref_res, k)) <= 2e-5 * cond, tag
    assert rel_l2(grads, ref_grads) <= 1e-4 * cond, tag
    check_tensors(spec, grads, ref_grads, 2e-4 * cond)
    assert u.shape == (pts.shape[0], k), tag
    assert rel_l2(u, prob.predict(pts.astype(np.float64)).reshape(-1, k)) <= 1e-5, tag


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_width_edge_matches_fp64_oracle(case):
    _, seed, fixed = case
    cfg, prob, params, pts, (_, _, _, r64, thr), spec = random_setup(seed, kind='mse', n=N_POINTS, **fixed)
    got = EC.emul_coupled_step(spec, params, pts)
    check_against_oracle(cfg, prob, spec, pts, got, EC.emul_coupled_forward(spec, params, pts), r64, thr)


def test_cases_cover_the_edges():
    """ what the cases claim to reach, from the specs they build """
    setups = [(c[0], random_setup(c[1], kind='mse', n=1, **c[2])) for c in CASES]
    specs = [s[-1] for _, s in setups]
    hidden = lambda s: [s.widths[l] for l in range(1, s.n_layers)]
    assert {(s.nf, s.ns) for s in specs} == set(JET_SETS)
    assert {s.widths[s.n_layers] for s in specs} == {2, 3, 4}
    assert set(EDGE_WIDTHS) <= {w for s in specs for w in hidden(s)}
    assert any(s.skip_src[l] >= 0 for s in specs for l in range(s.n_layers) if max(hidden(s)) >= 64)   # a wide residual net
    # the output layer's n_in on another block edge than a hidden layer's width
    assert any(len(set((w + 1 + 7) // 8 for w in hidden(s))) > 1 for s in specs)
    assert any(s.n_vars == 2 and s.ic_has_vars and s.widths[s.n_layers] > 2 for s in specs)
    assert max(s.widths[0] for s in specs) == 8 and {6, 7, 8} <= {s.widths[0] for s in specs}
