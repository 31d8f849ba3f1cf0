""" The trained-state fixtures (tests/trained_state.py) and the host emulation of the device math held to their bar.

The fixtures are the parameters an fp64 fit reaches, with points on the faces, corners and time ends of the domain, in
three variants: as trained, with the hidden layers saturated, and with a sharp time gate.  Here: the fixtures reproduce
(the fp64 oracle at the stored parameters gives the stored results), each variant is what it claims to be, and the
g++ build of the per-thread device code (tests/emul) passes the bar of trained_state.check at every variant of every
problem the thread kernels run (the tensor-core tile kernels have no host twin; test_gpu_trained_state.py holds them
on the device).  The bar's floor F was set from these runs: the worst ratio |K - X| / max(|R - X|, F S) over all of
them stays below C. """
import numpy as np
import pytest
import torch

import trained_state as TS

NAMES = list(TS.FIXTURES)
EMULATED = [n for n in NAMES if not TS.FIXTURES[n][0].startswith('tile128')]
CASES = [(n, v) for n in NAMES for v in TS.variant_names(n)]
EMUL_CASES = [(n, v) for n, v in CASES if n in EMULATED]


@pytest.mark.parametrize('name', NAMES)
def test_fixture_reproduces(name):
    fx = TS.load(name)
    assert np.array_equal(fx['points'], TS.fixture_points(name))
    params, X = TS.fixture_variant(fx, name, 'trained')
    got = TS.evaluate(name, params, fx['points'])
    for key in ('residual', 'grads', 'u', 'S'):
        a, b = np.asarray(got[key]), np.asarray(X[key])
        assert np.linalg.norm(a - b) <= 1e-10 * np.linalg.norm(b), key
    assert abs(got['loss'] - X['loss']) <= 1e-10 * abs(X['loss'])


@pytest.mark.parametrize('name', NAMES)
def test_fit_reduced_the_loss(name):
    steps, lr, seed, batch, loss0, loss1 = TS.load(name)['meta']
    _, want_steps, want_batch, want_lr, want_seed = TS.FIXTURES[name]
    assert (int(steps), int(batch), lr, int(seed)) == (want_steps, want_batch, want_lr, want_seed), 'fixture out of date'
    assert loss1 * TS.min_drop(name) <= loss0, '%s: loss %.3e -> %.3e' % (name, loss0, loss1)


@pytest.mark.parametrize('name', NAMES)
def test_points_cover_faces_corners_and_time_ends(name):
    cfg, pts = TS.cfg_of(name), TS.load(name)['points']
    dom = TS.domain_of(name)
    nsp = cfg['ndims'] - 1 if TS.has_ic(name) else cfg['ndims']
    for i in range(nsp):
        for side in (0, 1):
            assert (pts[:, i] == np.float32(dom[i][side])).sum() >= TS.EDGE, (i, side)
    if nsp:
        corner = np.all([np.isin(pts[:, i], np.float32(dom[i])) for i in range(nsp)], axis=0)
        assert corner.sum() >= 2 ** nsp
    if TS.has_ic(name):
        t = cfg['ndims'] - 1
        assert (pts[:, t] == np.float32(dom[t][0])).sum() >= TS.EDGE
        assert (pts[:, t] == np.float32(cfg['ranges'][t][1])).sum() >= TS.EDGE
    if nsp:
        interior = np.all([(pts[:, i] > dom[i][0]) & (pts[:, i] < dom[i][1]) for i in range(nsp)], axis=0)
        assert interior.sum() >= TS.N_POINTS // 2


@pytest.mark.parametrize('name', NAMES)
def test_saturated_variant_saturates_every_hidden_layer_but_the_first(name):
    fx = TS.load(name)
    zs = TS.pre_activations(name, TS.variant_params(name, fx['trained'], 'saturated'), fx['points'])
    for l, z in enumerate(zs[1:], 1):
        share = float((np.abs(z) > 3).mean())
        assert share >= 0.3, '%s: hidden layer %d has %.0f %% of |z| > 3' % (name, l, 100 * share)


@pytest.mark.parametrize('name', [n for n in NAMES if TS.has_ic(n)])
def test_sharp_gate_saturates_the_time_gate(name):
    fx = TS.load(name)
    cfg = TS.cfg_of(name)
    p = TS.variant_params(name, fx['trained'], 'sharp_gate')
    t = fx['points'][:, cfg['ndims'] - 1].astype(np.float64)
    w = (t - TS.domain_of(name)[-1][0]) / np.exp(float(p[dict(TS.tensors(name))['log_scale']][0]))
    assert (np.abs(w) > 5).mean() >= 0.5
    assert (w == 0).sum() >= TS.EDGE                    # and the points at t = t0, where the gate is 0 and its slope 1/4


def emulate(name, params, pts):
    """ the host emulation of the thread kernels' step and forward -> dict(loss, residual, grads, u) """
    spec = TS.spec_of(name)
    if 'k' in TS.cfg_of(name):
        import emul_coupled as EC
        loss, res, grads = EC.emul_coupled_step(spec, params, pts)
        u = EC.emul_coupled_forward(spec, params, pts)
    else:
        import emul_harness as E
        loss, res, grads = E.emul_step(spec, params, pts)
        u = E.emul_forward(spec, params, pts)
    return dict(loss=loss, residual=res, grads=grads, u=u)


_R = {}


def fp32_oracle(name, variant, params, pts):
    """ the fp32 oracle (R of the bar) on the whole batch at once, kept per problem and variant """
    if (name, variant) not in _R:
        _R[(name, variant)] = TS.evaluate(name, params, pts, dtype=torch.float32, chunks=1)
    return _R[(name, variant)]


@pytest.mark.parametrize('name,variant', EMUL_CASES)
def test_host_emulation_passes_the_bar(name, variant):
    fx = TS.load(name)
    params, X = TS.fixture_variant(fx, name, variant)
    K = emulate(name, params, fx['points'])
    R = fp32_oracle(name, variant, params, fx['points'])
    worst = TS.check('emulation %s %s %s' % (TS.FIXTURES[name][0], variant, name), name, K, R, X)
    print('WORST %s %s %.3f' % (name, variant, worst))
