""" FusedEngine — host side of the fused fit step: flat parameter/gradient buffers, the plan, the
per-step launch sequence and its CUDA-graph capture, data-parallel sharding.

Per step (replaces reference pydens/model_torch.py:427-464):
    pinn_step         sample + forward jets + residual + MSE + backward     (one CUDA kernel); with
                      torch.distributed initialised: pinn_step_allreduce, whose tail sums [grads | loss] over
                      the ranks through NVLink peer memory (NCCL all_reduce only if IPC mapping is unavailable)
    constraints       one more launch of the same kernel family per lowered constraint, added to [grads | loss]
                      (constraints that do not lower are added by autograd)
    optimizer.step()  torch (fused, capturable Adam by default) on views of the flat buffer
    pinn_record_loss  loss -> device ring, advance the device step counter
The sequence is captured once in a CUDA graph and replayed; nothing in it touches the host.
"""
import ctypes as C
import os
import warnings

import numpy as np
import torch

from . import _native
from .solver import _progress

_GRAPH_MIN_ITERS = 8
_HOST_GRAPH_MIN_ITERS = 8           # host-sampler mode: one capture per staging buffer
_AUTO_PERSISTENT_STEPS = 50         # optimizer steps per launch when a tiny-batch fit goes to the persistent kernel by itself
_AUTO_PERSISTENT_MIN_ITERS = 16
_RING_LEN = 1 << 15                 # device loss ring (steps between two read-backs of a long fit)


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist
    return None


def capture_graph(device, body, pool=None):
    """ Capture `body()` into a CUDA graph on a side stream.  Unlike the `torch.cuda.graph` context manager this
    does not run the garbage collector and does not empty the allocator cache, which is what makes a capture
    cost ~20 ms there; a fit only pays a millisecond or two here. """
    import gc
    _reap()                                          # native objects whose teardown was postponed: now is a safe moment
    graph = torch.cuda.CUDAGraph()
    current = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device=device)
    side.wait_stream(current)
    # the collector must not run finalizers while the capture is open: an old engine's __del__ frees device memory
    # and synchronises streams, which is illegal during a (global-mode) capture and invalidates it
    gc_was_enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.stream(side):
            try:
                # thread-local error mode: other threads (the NCCL watchdog polling its events when the NCCL fallback
                # all-reduce is part of the step) may keep calling into CUDA while this thread captures
                if pool is not None:
                    graph.capture_begin(pool=pool, capture_error_mode='thread_local')
                else:
                    graph.capture_begin(capture_error_mode='thread_local')
                body()
                graph.capture_end()
            except Exception:
                try:
                    graph.capture_end()
                except Exception:                       # noqa: BLE001
                    pass
                raise
    finally:
        if gc_was_enabled:
            gc.enable()
    current.wait_stream(side)
    return graph


_graveyard = []                                      # (destroy function, handle) postponed because a capture was open


def _capturing():
    try:
        return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()
    except Exception:                                # noqa: BLE001
        return False


def _destroy(fn, handle):
    """ Tear a native object down now, or — inside a stream capture, where freeing device memory is illegal — later. """
    if _capturing():
        _graveyard.append((fn, handle))
    else:
        fn(handle)


def _reap():
    if _graveyard and not _capturing():
        pending, _graveyard[:] = list(_graveyard), []
        for fn, handle in pending:
            fn(handle)


def shard_batch(batch_size, world, rank):
    """ Contiguous, near-equal split of the global batch over ranks -> (local_n, point_offset).
    The Philox counter is the GLOBAL point index, so the sampled batch does not depend on `world`. """
    base, rem = divmod(int(batch_size), int(world))
    return base + (1 if rank < rem else 0), rank * base + min(rank, rem)


def sampler_columns(sampler, total):
    """ Where a sampler's batches come from: (key, cols) with `cols` its in-kernel columns (None: the kernels' uniform
    default) and `key` equal for samplers that draw the same columns, or (None, None): sampled on the host. """
    if sampler is None:
        return 'uniform', None
    dev_cols = sampler.device_columns() if hasattr(sampler, 'device_columns') else None
    if dev_cols is not None and len(dev_cols) == total and os.environ.get('PYDENS_B200_HOST_SAMPLER') != '1':
        try:
            cols = _native.make_columns(dev_cols, total)
            return bytes(cols), cols
        except ValueError:                    # more mixture components than the kernel takes
            pass
    return None, None


def plain_adam(opt):
    """ The optimizer is the Adam the kernels implement: torch.optim.Adam, one parameter group, no amsgrad, no
    maximize, a float lr, and weight decay added to the gradient (L2).  Adam(decoupled_weight_decay=True) is AdamW,
    which the kernels do not implement; with zero weight decay both forms are the same update. """
    g = opt.param_groups[0] if opt.param_groups else {}
    return (type(opt) is torch.optim.Adam and len(opt.param_groups) == 1 and not g.get('amsgrad')
            and not g.get('maximize') and not torch.is_tensor(g.get('lr'))
            and not (g.get('decoupled_weight_decay') and g.get('weight_decay')))


def adam_steps_equal(opt):
    """ Every parameter of the optimizer has taken the same number of steps (a parameter without state: none).  torch
    keeps one step count per tensor, the kernels take one t for all of them; a state loaded with differing counts runs
    on torch's Adam. """
    steps = {float(st['step']) if st and 'step' in st else 0.0
             for st in (opt.state.get(p) for g in opt.param_groups for p in g['params'])}
    return len(steps) <= 1


def adam_hyper(opt):
    """ (lr, (beta1, beta2), eps, weight_decay) of a plain_adam optimizer """
    g = opt.param_groups[0]
    return float(g['lr']), tuple(map(float, g['betas'])), float(g['eps']), float(g['weight_decay'])


def auto_persistent(niters, batch_size, info):
    """ A fit goes to the persistent kernels without steps_per_launch: tiny batches (launch- and latency-bound one step
    at a time) and enough steps.  PYDENS_B200_AUTO_PERSISTENT=0 keeps one launch per step. """
    return (niters >= _AUTO_PERSISTENT_MIN_ITERS and 0 < batch_size <= int(info.small_batch_points)
            and os.environ.get('PYDENS_B200_AUTO_PERSISTENT', '1') != '0' and os.environ.get('PYDENS_B200_NO_GRAPH') != '1')


def ring_losses(ring, start, lo, hi):
    """ The losses of steps [lo, hi) of a fit whose first step went to ring entry `start` (modulo the ring's length),
    read from the device loss ring; the caller has synchronised the device. """
    return ring.cpu().numpy()[(start + np.arange(lo, hi)) % ring.numel()]


def _term_array(terms, total_sum):
    """ The constraint terms of a persistent fit as a PinnTerm array, with their point weights: the mean of
    model_torch.py:448 over every constraint's own points, or 1 for reduction='sum'. """
    term_arr = (_native.PinnTerm * max(1, len(terms)))()
    for i, e in enumerate(terms):
        term_arr[i].plan = e['plan'].value
        term_arr[i].n_points = e['n']
        term_arr[i].point_weight = 1.0 if total_sum else 1.0 / e['n']
        term_arr[i].points = e['host_points'].data_ptr()
    return term_arr


def _persistent_launches(engines, samplers, niters, batch_size, k, members, launch):
    """ The launch loop of a persistent fit: `niters` steps of every engine's fit, at most `k` (and the loss ring's
    length) per launch.  For host samplers each member's batches of a launch are staged on the device and set in its
    row of `members` (a ctypes array whose rows have `points`); `launch(done, kk)` then issues the launches of steps
    done .. done + kk - 1 and returns None, or the library's message when it refused the first launch with
    PINN_E_UNSUPPORTED (no step has been taken then: returned as it is).  The losses of every step are read from the
    device rings and appended to each solver's `losses`; `steps_done` advances. """
    e0 = engines[0]
    total, ring_len = e0.solver.model.total, e0.ring.numel()
    host = sampler_columns(samplers[0], total)[0] is None
    starts = [eng.steps_done for eng in engines]
    vals = np.empty((len(engines), niters), dtype=np.float32)

    def drain(lo, hi):
        torch.cuda.synchronize(e0.device)
        for j, eng in enumerate(engines):
            vals[j, lo:hi] = ring_losses(eng.ring, starts[j], lo, hi)

    done, drained = 0, 0
    while done < niters:
        kk = min(k, niters - done, ring_len)
        if done + kk - drained > ring_len:
            drain(drained, done)
            drained = done
        batches = []                                      # each member's kk batches, alive until the launch
        if host:
            for mb, smp in zip(members, samplers):
                pinned = torch.empty((kk, batch_size, total), dtype=torch.float32).pin_memory()
                for i in range(kk):
                    b = smp.sample(batch_size)
                    pinned[i].copy_(b if isinstance(b, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32)))
                batches.append(pinned.to(e0.device, non_blocking=True))
                mb.points = batches[-1].data_ptr()
        refused = launch(done, kk)
        if refused is not None:
            return refused
        done += kk
    drain(drained, niters)
    for j, eng in enumerate(engines):
        eng.steps_done = starts[j] + niters
        eng.solver.losses.extend(np.array(x, dtype=np.float32) for x in vals[j])
    return None


def _first_refusal(rc, lib, done, lo):
    """ The library's message when it refused the first launch of a fit as unsupported, else None (raises on other
    errors). """
    if rc == _native.E_UNSUPPORTED and done == 0 and lo == 0:
        return lib.pinn_last_error().decode('utf-8', 'replace')
    _native.check(rc)
    return None


def run_persistent(engines, opts, samplers, terms, niters, batch_size, k, table):
    """ `niters` optimizer steps of every engine's fit, `k` per launch of the persistent multi-step kernels: the
    reference loop model_torch.py:426-464 with optimizer.step() inside the kernel, constraint terms included.  One fit
    runs on the solo kernels (pinn_multi_step_terms) unless `table` is set; with `table` the fits are members of
    pinn_multi_step_ensemble_adam, at most MAX_MEMBERS per launch, each with the Adam hyper-parameters of its own
    optimizer.  `samplers` has one sampler per fit: all in-kernel with the same columns, or all on the host.  Returns
    None, or the library's message when it refused the first launch with PINN_E_UNSUPPORTED (no step has been taken
    then). """
    e0 = engines[0]
    lib, total, ring_len = e0.lib, e0.solver.model.total, e0.ring.numel()
    total_sum = e0._sum_reduction()
    term_arr = _term_array(terms, total_sum)
    point_weight = 1.0 if total_sum else 1.0 / batch_size
    M = len(engines)
    members = (_native.PinnMember * M)()
    hyper = (_native.PinnAdamHyper * M)()
    step0 = []
    for mb, hy, eng, opt in zip(members, hyper, engines, opts):
        hy.lr, (hy.beta1, hy.beta2), hy.eps, hy.weight_decay = adam_hyper(opt)
        eng._adopt_optimizer()
        mask = eng._bind_adam_state(opt)
        m, v, steps, _ = eng._adam_flat
        mb.params, mb.exp_avg, mb.exp_avg_sq, mb.mask = eng.flat.data_ptr(), m.data_ptr(), v.data_ptr(), mask.data_ptr()
        mb.step_tensors, mb.n_step_tensors = steps.data_ptr(), steps.numel()
        mb.seed, mb.step_counter, mb.losses_ring = eng.seed, eng.step_counter.data_ptr(), eng.ring.data_ptr()
        step0.append(float(steps.max().item()))
        eng.solver.model.train()
    cols = sampler_columns(samplers[0], total)[1]
    lr, (b1, b2), eps, wd = adam_hyper(opts[0])
    stream = e0._stream()
    size, hsize = C.sizeof(_native.PinnMember), C.sizeof(_native.PinnAdamHyper)

    def launch(done, kk):
        for mb, s0 in zip(members, step0):
            mb.opt_step0 = s0 + done
        for lo in range(0, M, _native.MAX_MEMBERS):
            if table:
                rc = lib.pinn_multi_step_ensemble_adam(
                    e0.plan, min(_native.MAX_MEMBERS, M - lo),
                    C.cast(C.addressof(members) + lo * size, C.POINTER(_native.PinnMember)),
                    C.cast(C.addressof(hyper) + lo * hsize, C.POINTER(_native.PinnAdamHyper)), C.c_int64(batch_size),
                    C.c_int(kk), C.c_int64(ring_len), C.c_float(point_weight), C.c_int(len(terms)), term_arr, cols,
                    stream)
            else:
                mb = members[0]
                rc = lib.pinn_multi_step_terms(
                    e0.plan, mb.params, mb.exp_avg, mb.exp_avg_sq, mb.mask, mb.step_tensors, mb.n_step_tensors,
                    mb.points, cols, mb.seed, mb.step_counter, C.c_int64(batch_size), C.c_int(kk), C.c_float(lr),
                    C.c_float(b1), C.c_float(b2), C.c_float(eps), C.c_float(wd), C.c_float(mb.opt_step0),
                    mb.losses_ring, C.c_int64(ring_len), C.c_float(point_weight), C.c_int(len(terms)), term_arr, stream)
            refused = _first_refusal(rc, lib, done, lo)
            if refused is not None:
                return refused
        return None

    return _persistent_launches(engines, samplers, niters, batch_size, k, members, launch)


def run_lbfgs_persistent(engines, opts, samplers, terms, niters, batch_size, k, table):
    """ `niters` L-BFGS steps of every engine's fit, `k` per launch of the L-BFGS form of the cluster kernel: every
    evaluation of a step and the update between them run in the kernel, on the step's one batch, with the constraint
    terms.  One fit runs through pinn_lbfgs_multi unless `table` is set; with `table` the fits are members of
    pinn_lbfgs_multi_ensemble, at most MAX_MEMBERS per launch, each with its own lr and frozen mask and the other
    settings of opts[0].  Each device state is bound as _fit_lbfgs binds it and written back into opt.state at the end.
    Returns None, or the library's message when it refused the first launch with PINN_E_UNSUPPORTED (no step has been
    taken then). """
    e0 = engines[0]
    lib, total = e0.lib, e0.solver.model.total
    total_sum = e0._sum_reduction()
    term_arr = _term_array(terms, total_sum)
    point_weight = 1.0 if total_sum else 1.0 / batch_size
    M = len(engines)
    members = (_native.PinnLbfgsMember * M)()
    binds = []
    for mb, eng, opt in zip(members, engines, opts):
        eng._adopt_optimizer()
        cfg, cur, mask = eng._lbfgs_bind(opt)
        binds.append((cfg, cur, mask))
        mb.params, mb.state, mb.mask = eng.flat.data_ptr(), cur['state'].data_ptr(), mask.data_ptr()
        mb.seed, mb.step_counter, mb.losses_ring, mb.lr = eng.seed, eng.step_counter.data_ptr(), eng.ring.data_ptr(), cfg.lr
        eng.solver.model.train()
    cfg = binds[0][0]
    cols = sampler_columns(samplers[0], total)[1]
    stream = e0._stream()
    size = C.sizeof(_native.PinnLbfgsMember)

    def launch(done, kk):
        for lo in range(0, M, _native.MAX_MEMBERS):
            if table:
                rc = lib.pinn_lbfgs_multi_ensemble(
                    e0.plan, C.byref(cfg), min(_native.MAX_MEMBERS, M - lo),
                    C.cast(C.addressof(members) + lo * size, C.POINTER(_native.PinnLbfgsMember)), cols,
                    C.c_int64(batch_size), C.c_int(kk), C.c_float(point_weight), C.c_int(len(terms)), term_arr, stream)
            else:
                mb = members[0]
                rc = lib.pinn_lbfgs_multi(e0.plan, C.byref(cfg), mb.params, mb.state, mb.points, cols, mb.seed,
                                          C.c_int64(batch_size), C.c_int(kk), C.c_float(point_weight),
                                          C.c_int(len(terms)), term_arr, stream)
            refused = _first_refusal(rc, lib, done, lo)
            if refused is not None:
                return refused
        return None

    refused = _persistent_launches(engines, samplers, niters, batch_size, k, members, launch)
    if refused is None:
        for eng, opt, (_, cur, _) in zip(engines, opts, binds):
            cur['fresh'] = lbfgs_export(cur['state'], opt, cur['idx'], eng.n_params, cur['m'])
    return refused


class FusedEngine:
    def __init__(self, solver):
        self.lib = _native.load()
        self.solver = solver
        model, traced, chain = solver.model, solver._traced, solver._chain
        self.device = solver.device
        if self.device.type != 'cuda':
            raise RuntimeError('the fused engine needs a CUDA device (got %s); there is no CPU fallback' % self.device)
        torch.cuda.set_device(self.device)

        # ---- canonical flat layout: W_0, b_0, ..., log_scale, equation variables, everything else ----
        entries, off = [], 0
        w_off, b_off = [], []
        for lin, _, _ in chain:
            w_off.append(off); entries.append((lin.weight, off)); off += lin.weight.numel()
            b_off.append(off); entries.append((lin.bias, off)); off += lin.bias.numel()
        log_scale_off = off
        entries.append((model.log_scale, off)); off += 1
        var_offsets = {}
        for name in traced.var_names:
            p = getattr(model, name)
            var_offsets[name] = off
            entries.append((p, off)); off += p.numel()
        seen = {id(p) for p, _ in entries}
        for p in model.parameters():
            if id(p) not in seen:
                entries.append((p, off)); off += p.numel(); seen.add(id(p))
        self.n_params = (off + 3) // 4 * 4
        self.entries = entries
        self.flat = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
        self.out = torch.zeros(self.n_params + 4, dtype=torch.float32, device=self.device)
        with torch.no_grad():
            for p, o in entries:
                n = p.numel()
                self.flat[o:o + n].copy_(p.data.reshape(-1).to(torch.float32))
                p.data = self.flat[o:o + n].view(p.shape)
                p.grad = self.out[o:o + n].view(p.shape)

        widths = [model.total] + [c[0].out_features for c in chain]
        acts = [c[1] for c in chain]
        skips = [c[2] for c in chain]
        has_bc = model.boundary_condition is not None
        has_ic = model.raw_initial_condition is not None
        self._spec_args = (widths, acts, model.ndims, model.nparams, has_bc,
                           model.boundary_condition if has_bc else 0.0, has_ic, model.domain)
        self._spec_kwargs = dict(var_offsets=var_offsets, w_off=w_off, b_off=b_off, log_scale_off=log_scale_off,
                                 n_params=self.n_params, skips=skips)
        self.spec = _native.build_spec(*self._spec_args, traced, **self._spec_kwargs)
        self._constraint_plans = {}                       # num -> fused constraint launch (see _constraint_plan)
        plan = C.c_void_p()
        _native.check(self.lib.pinn_plan_create(C.byref(self.spec), self.device.index, C.byref(plan)))
        self.plan = plan
        self.info = _native.PinnPlanInfo()
        _native.check(self.lib.pinn_plan_info(self.plan, C.byref(self.info)))
        ws_bytes = self.lib.pinn_workspace_bytes(self.plan, 1)
        self.workspace = torch.zeros(ws_bytes, dtype=torch.uint8, device=self.device)
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.ring = torch.zeros(_RING_LEN, dtype=torch.float32, device=self.device)
        self.steps_done = 0
        self._graphs, self._pipes, self._pinned_batches = {}, {}, {}
        self._opt_obj, self._opt_key, self._loss_host = None, None, None
        self._adam_flat = None
        self._adam_bound_to, self._adam_bound_sig = None, None
        self.seed = solver.seed

        self.comm = None
        dist = _dist()
        if dist is not None:
            seed_t = torch.tensor([self.seed], dtype=torch.int64, device=self.device)
            dist.broadcast(seed_t, 0)
            self.seed = int(seed_t.item())
            dist.broadcast(self.flat, 0)
            self._connect_peers(dist)

    def _connect_peers(self, dist):
        """ Set up the in-kernel all-reduce over NVLink peer memory (pinn_step_allreduce): every rank
        allocates an exchange buffer inside the library, the CUDA-IPC handles are gathered and mapped.
        Any failure (no peer access, more than 8 ranks, several nodes) leaves NCCL in charge. """
        if os.environ.get('PYDENS_B200_FUSED_ALLREDUCE', '1') == '0':
            return
        world, rank = dist.get_world_size(), dist.get_rank()
        ok, comm = 1, C.c_void_p()
        handle = (C.c_ubyte * 64)()
        if world > 8 or self.lib.pinn_comm_create(self.plan, rank, world, C.byref(comm), handle) != 0:
            ok = 0
        handles = [None] * world
        dist.all_gather_object(handles, bytes(handle) if ok else None)
        if ok and all(h is not None for h in handles):
            ok = int(self.lib.pinn_comm_connect(comm, b''.join(handles)) == 0)
        else:
            ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=self.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)              # all ranks or none
        if int(flag.item()) == 1:
            self.comm = comm
        elif comm:
            self.lib.pinn_comm_destroy(comm)

    def __del__(self):
        try:
            self._drop_graphs()
            if getattr(self, 'comm', None):
                _destroy(self.lib.pinn_comm_destroy, self.comm)
                self.comm = None
            for entry in getattr(self, '_constraint_plans', {}).values():
                if entry is not None and entry.get('plan'):
                    self.lib.pinn_plan_destroy(entry['plan'])
                    entry['plan'] = None
            if getattr(self, 'plan', None):
                self.lib.pinn_plan_destroy(self.plan)
                self.plan = None
        except Exception:                                  # pragma: no cover
            pass

    def _constraint_plan(self, num):
        """ Constraint `num` as one more launch of the same kernel family (reference :451-457): a plan whose
        residual program is the traced constraint (on its own jet set or the equation's), run on the constraint's own points
        with 1/n weighting; its [grads | loss] buffer is then added to the step's.  None -> autograd adds it. """
        if num not in self._constraint_plans:
            entry = None
            lowered = self.solver._lower_constraint(num)
            if lowered is not None:
                traced, pts = lowered
                spec = _native.build_spec(*self._spec_args, traced, **self._spec_kwargs)
                plan = C.c_void_p()
                rc = self.lib.pinn_plan_create(C.byref(spec), self.device.index, C.byref(plan))
                if rc == 0:
                    ws = torch.zeros(self.lib.pinn_workspace_bytes(plan, 1), dtype=torch.uint8, device=self.device)
                    entry = dict(plan=plan, spec=spec, points=pts.to(self.device).contiguous(), n=int(pts.shape[0]),
                                 out=torch.zeros(self.n_params + 4, dtype=torch.float32, device=self.device),
                                 workspace=ws, host_points=pts.detach().cpu().contiguous())
                elif rc != _native.E_UNSUPPORTED:
                    _native.check(rc)
            self._constraint_plans[num] = entry
        return self._constraint_plans[num]

    def _constraint_step(self, entry):
        _native.check(self.lib.pinn_step(
            entry['plan'], C.c_void_p(self.flat.data_ptr()), C.c_void_p(entry['points'].data_ptr()), None,
            C.c_uint64(self.seed), None, C.c_uint64(0), C.c_uint64(0), C.c_int64(entry['n']),
            C.c_float(1.0 if self._sum_reduction() else 1.0 / entry['n']), C.c_void_p(entry['out'].data_ptr()), None,
            C.c_void_p(entry['workspace'].data_ptr()), C.c_size_t(entry['workspace'].numel()), self._stream()))
        self.out.add_(entry['out'])                       # [grads | loss] += the constraint's

    def _sum_reduction(self):
        """ criterion(reduction='sum') of the fit this engine was built for (Solver._crit_key ends with 'sum') """
        return getattr(self.solver, '_crit_key', ('mse',))[-1] == 'sum'

    def release(self):
        """ Give every parameter its own storage back (the autograd path is taking over). """
        with torch.no_grad():
            for p, _ in self.entries:
                p.data = p.data.clone()
                p.grad = None

    # ------------------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _step(self, points, cols, n_points, inv_n, point_offset, residual=None, use_counter=True, step_value=0,
              allreduce=False):
        args = (C.c_void_p(self.flat.data_ptr()),
                C.c_void_p(points.data_ptr()) if points is not None else None,
                cols, C.c_uint64(self.seed),
                C.c_void_p(self.step_counter.data_ptr()) if use_counter else None, C.c_uint64(step_value),
                C.c_uint64(point_offset), C.c_int64(n_points), C.c_float(inv_n),
                C.c_void_p(self.out.data_ptr()),
                C.c_void_p(residual.data_ptr()) if residual is not None else None,
                C.c_void_p(self.workspace.data_ptr()), C.c_size_t(self.workspace.numel()), self._stream())
        if allreduce and self.comm is not None:
            _native.check(self.lib.pinn_step_allreduce(self.plan, self.comm, *args))
        else:
            _native.check(self.lib.pinn_step(self.plan, *args))

    def _step_adam(self, points, cols, n_points, inv_n, point_offset, adam, allreduce=False):
        """ The whole step in ONE launch (pinn_step_adam): kernel -> in-kernel all-reduce -> Adam -> loss log. """
        _native.check(self.lib.pinn_step_adam(
            self.plan, self.comm if (allreduce and self.comm is not None) else None,
            C.c_void_p(self.flat.data_ptr()), C.c_void_p(points.data_ptr()) if points is not None else None,
            cols, C.c_uint64(self.seed), C.c_void_p(self.step_counter.data_ptr()), C.c_uint64(point_offset),
            C.c_int64(n_points), C.c_float(inv_n), C.c_void_p(self.out.data_ptr()), None,
            C.c_void_p(self.workspace.data_ptr()), C.c_size_t(self.workspace.numel()), C.byref(adam), self._stream()))

    def loss_and_grads(self, points):
        pts = torch.as_tensor(points, dtype=torch.float32).to(self.device).contiguous()
        n = pts.shape[0]
        residual = torch.empty(n, dtype=torch.float32, device=self.device)
        self._step(pts, None, n, 1.0 / n, 0, residual=residual, use_counter=False)
        torch.cuda.synchronize(self.device)
        return float(self.out[self.n_params].item()), self.out[:self.n_params].clone(), residual

    def sample(self, n_points, cols=None, step=None, point_offset=0):
        """ The batch the in-kernel sampler produces (tests / replay). """
        total = self.solver.model.total
        out = torch.empty((n_points, total), dtype=torch.float32, device=self.device)
        arr = _native.make_columns(cols, total)
        _native.check(self.lib.pinn_sample(
            self.plan, arr, C.c_uint64(self.seed),
            C.c_void_p(self.step_counter.data_ptr()) if step is None else None,
            C.c_uint64(0 if step is None else step), C.c_uint64(point_offset), C.c_int64(n_points),
            C.c_void_p(out.data_ptr()), self._stream()))
        return out

    def forward(self, pts):
        """ u at explicit points: [n] for a network of one output, [n, k] (row-major) for k outputs. """
        pts = pts.to(self.device, torch.float32).contiguous()
        n = pts.shape[0]
        k = self.solver._traced.n_out
        u = torch.empty((n, k) if k > 1 else n, dtype=torch.float32, device=self.device)
        _native.check(self.lib.pinn_forward(self.plan, C.c_void_p(self.flat.data_ptr()), C.c_void_p(pts.data_ptr()),
                                            C.c_int64(n), C.c_void_p(u.data_ptr()),
                                            C.c_void_p(self.workspace.data_ptr()),
                                            C.c_size_t(self.workspace.numel()), self._stream()))
        return u

    # ------------------------------------------------------------------------------------------
    def _optimizer_for(self, optimizer, lr, kwargs):
        """ The optimizer of this fit.  The reference builds a NEW optimizer on every `fit` (model_torch.py:419-422);
        a fresh fused Adam differs from a used one only by its state, so when the request repeats the previous one
        exactly, the existing object is kept and its state is zeroed in place — which keeps the captured CUDA graphs
        (they hold pointers into that state) valid across `fit` calls.  Returns (optimizer, state_is_materialised). """
        solver = self.solver
        if optimizer is None:
            solver._make_optimizer(None, lr)
            return solver.optimizer, bool(solver.optimizer.state)
        params = [p for p in solver.model.parameters() if p.requires_grad]
        key = (optimizer, float(lr), tuple(sorted((k, repr(v)) for k, v in kwargs.items())), tuple(id(p) for p in params))
        prev = solver.optimizer
        if (prev is not None and prev is self._opt_obj and key == self._opt_key and optimizer in ('Adam', 'AdamW')
                and prev.state and not any(kwargs.get(k) for k in ('amsgrad', 'maximize'))):
            with torch.no_grad():
                bound = self._adam_flat is not None and self._adam_bound_to is prev
                if bound:                                   # the state tensors are views of three flat buffers: three launches
                    spans = []
                    for buf in self._adam_flat[:3]:
                        buf.zero_()
                        spans.append((buf.data_ptr(), buf.data_ptr() + 4 * buf.numel()))
                    for st in prev.state.values():          # ... plus whatever state lives elsewhere
                        for v in st.values():
                            if torch.is_tensor(v) and not any(a <= v.data_ptr() < e for a, e in spans):
                                v.zero_()
                else:
                    for st in prev.state.values():
                        for v in st.values():
                            if torch.is_tensor(v):
                                v.zero_()
            return prev, True
        self._drop_graphs()
        solver._make_optimizer(optimizer, lr, fused_hint=True, **kwargs)
        self._opt_obj, self._opt_key = solver.optimizer, key
        return solver.optimizer, False

    def _adopt_optimizer(self):
        """ The solver's optimizer was not built by _optimizer_for (optimizer=None with an optimizer built elsewhere):
        the captured graphs hold pointers into another optimizer's state, and no request matches this one. """
        if self.solver.optimizer is not self._opt_obj:
            self._drop_graphs()
            self._opt_obj, self._opt_key = self.solver.optimizer, None

    def _drop_graphs(self):
        self._graphs = {}
        for pipe in getattr(self, '_pipes', {}).values():
            _destroy(self.lib.pinn_pipe_destroy, pipe)
        self._pipes = {}

    def _pinned_losses(self, n):
        if self._loss_host is None or self._loss_host.numel() < n:
            self._loss_host = torch.zeros(max(n, 4096), dtype=torch.float32).pin_memory()
        return self._loss_host

    def _bind_adam_state(self, opt):
        """ Make the optimizer's per-parameter Adam state views of three flat buffers (moments in parameter layout,
        step counters side by side), so that the persistent multi-step kernel and torch's own `opt.step()` update
        the very same memory.  -> mask of trainable entries. """
        if self._adam_flat is None:
            self._adam_flat = (torch.zeros(self.n_params, dtype=torch.float32, device=self.device),
                               torch.zeros(self.n_params, dtype=torch.float32, device=self.device),
                               torch.zeros(len(self.entries), dtype=torch.float32, device=self.device),
                               torch.zeros(self.n_params, dtype=torch.float32, device=self.device))
        m, v, steps, mask = self._adam_flat
        in_opt = {id(q) for g in opt.param_groups for q in g['params']}
        sig = (id(opt), tuple(sorted(in_opt)))

        def bound(st, idx, o):
            # all three state tensors are still the views: load_state_dict keeps a moment that is already on the device
            # and replaces a step given on the host, so one of them alone says nothing about the others
            return (st is not None and 'exp_avg' in st and st['exp_avg'].data_ptr() == m.data_ptr() + 4 * o
                    and st['exp_avg_sq'].data_ptr() == v.data_ptr() + 4 * o and torch.is_tensor(st['step'])
                    and st['step'].data_ptr() == steps.data_ptr() + 4 * idx)
        if self._adam_bound_to is opt and self._adam_bound_sig == sig and all(
                bound(opt.state.get(p), idx, o) for idx, (p, o) in enumerate(self.entries) if id(p) in in_opt):
            return mask                                 # same optimizer, same parameters, still bound: nothing to do
        mask.zero_()
        rebound = False
        with torch.no_grad():
            for idx, (p, o) in enumerate(self.entries):
                n = p.numel()
                if id(p) not in in_opt:
                    continue
                mask[o:o + n] = 1.0
                st = opt.state.get(p)
                mv, vv = m[o:o + n].view(p.shape), v[o:o + n].view(p.shape)
                if st and 'exp_avg' in st:
                    if bound(st, idx, o):
                        continue
                    mv.copy_(st['exp_avg']); vv.copy_(st['exp_avg_sq']); steps[idx] = float(st['step'])
                else:
                    mv.zero_(); vv.zero_(); steps[idx] = 0.0
                opt.state[p] = {'step': steps[idx], 'exp_avg': mv, 'exp_avg_sq': vv}
                rebound = True
        if rebound:
            self._drop_graphs()                 # captured steps still point at the previous state tensors
        self._adam_bound_to, self._adam_bound_sig = opt, sig
        return mask

    def _persistent_terms(self, loss_terms, batch_size):
        """ The constraint terms of a fit as terms of the persistent kernels (pinn_multi_step_terms): a list of
        constraint plans, or None when the fit has no equation term, or a constraint that does not lower to a fused
        plan, or more terms / constraint points than the kernels take. """
        if 'equation' not in loss_terms:
            return None
        nums = self.solver._constraint_numbers(loss_terms)
        entries = [self._constraint_plan(n) for n in nums]
        if any(e is None for e in entries) or len(entries) > _native.MAX_TERMS:
            return None
        # the kernels run a term's program on the equation's jets: its plan carries no directions, or the same ones
        eq = self.solver._traced
        for n in nums:
            tr = self.solver._lower_constraint(n)[0]
            if tr.nf and (tr.order != 2 or eq.order != 2 or (tr.dirs, tr.dir_vecs, tr.ns) != (eq.dirs, eq.dir_vecs, eq.ns)):
                return None
        if sum(e['n'] for e in entries) > _native.MAX_TERM_POINTS:
            return None
        if batch_size + sum(e['n'] for e in entries) > self.lib.pinn_multi_step_max_points(self.plan):
            return None
        return entries

    def _lbfgs_persistent_terms(self, niters, batch_size, loss_terms, opt, steps_per_launch):
        """ The constraint terms of an L-BFGS fit that runs in the cluster kernel (run_lbfgs_persistent), or None when
        it does not: a plan without the cluster kernel, several ranks, an optimizer over parameters outside the fused
        network, constraints that do not all lower to persistent terms, a batch the kernel does not take, or a fit the
        rule of auto_persistent does not send there without steps_per_launch. """
        cap = int(self.info.small_batch_points)
        if niters <= 0 or batch_size <= 0 or not cap or _dist() is not None:
            return None
        if steps_per_launch <= 0 and not auto_persistent(niters, batch_size, self.info):
            return None
        g = opt.param_groups[0]
        entry_ids = {id(p) for p, _ in self.entries}
        if any(id(p) not in entry_ids for p in g['params']) or g['line_search_fn'] not in (None, 'strong_wolfe'):
            return None
        terms = self._persistent_terms(loss_terms, batch_size)
        if terms is None or batch_size + sum(e['n'] for e in terms) > cap:
            return None
        return terms

    def _fit_persistent(self, niters, batch_size, sampler, opt, k, terms=()):
        """ `niters` optimizer steps, `k` per launch of the solo persistent multi-step kernels (run_persistent).
        Returns False, having taken no step, when the kernels cannot hold the constraint programs' scratch slots. """
        refused = run_persistent([self], [opt], [sampler], terms, niters, batch_size, k, table=False)
        if refused is None:
            return True
        if terms:
            return False
        raise _native.NativeError(_native.E_UNSUPPORTED, refused)

    def fit(self, niters, batch_size, sampler, loss_terms, optimizer, criterion, lr, **kwargs):
        steps_per_launch = int(kwargs.pop('steps_per_launch', 0) or 0)
        opt, opt_ready = self._optimizer_for(optimizer, lr, kwargs)
        # Tiny batches (the README example: batch_size=100, niters=1500) are launch- and latency-bound one step at a
        # time: when nothing stands in the way, the loop runs in the persistent cluster kernel without being asked to,
        # _AUTO_PERSISTENT_STEPS optimizer steps per launch (same math, same loss log; PYDENS_B200_AUTO_PERSISTENT=0
        # keeps one launch per step).  An explicit steps_per_launch takes precedence.
        requested = steps_per_launch > 0
        if type(opt) is torch.optim.LBFGS and len(opt.param_groups) == 1:
            # tiny batches: every evaluation and update of a step in the L-BFGS form of the cluster kernel, by the same
            # rule as Adam's persistent fits
            terms = self._lbfgs_persistent_terms(niters, batch_size, loss_terms, opt, steps_per_launch)
            k = steps_per_launch if requested else _AUTO_PERSISTENT_STEPS
            if terms is not None and run_lbfgs_persistent([self], [opt], [sampler], terms, niters, batch_size, k,
                                                          table=False) is None:
                return
            if requested:
                warnings.warn('pydens_b200: steps_per_launch ignored (L-BFGS runs in the cluster kernel only on one '
                              'device, with fused constraints, over parameters of the fused network, for a batch of at '
                              'most %d points with the constraint points; otherwise one evaluation per launch)'
                              % int(self.info.small_batch_points), stacklevel=3)
            self._fit_lbfgs(niters, batch_size, sampler, loss_terms, criterion, opt)
            return
        if not requested and auto_persistent(niters, batch_size, self.info):
            steps_per_launch = _AUTO_PERSISTENT_STEPS
        if steps_per_launch > 0 and niters > 0:
            terms = None
            if plain_adam(opt) and adam_steps_equal(opt) and _dist() is None and batch_size > 0:
                terms = self._persistent_terms(loss_terms, batch_size)
            if terms is not None and self._fit_persistent(niters, batch_size, sampler, opt, steps_per_launch, terms):
                return
            if requested:
                warnings.warn('pydens_b200: steps_per_launch ignored (needs Adam, one device, the equation term, '
                              'constraints that run fused (at most %d, with %d points in all), batch + constraint points '
                              'of at most %d and a network that fits the persistent kernel)'
                              % (_native.MAX_TERMS, _native.MAX_TERM_POINTS,
                                 self.lib.pinn_multi_step_max_points(self.plan)), stacklevel=3)
        self._fit_stepwise(niters, batch_size, sampler, loss_terms, criterion, opt, opt_ready)

    def _eval_setup(self, niters, batch_size, sampler, loss_terms, criterion):
        """ What an evaluation of the objective (_evaluate) needs for a fit: the terms, this rank's share of the batch,
        the point weight, the sampler's columns; points every parameter's .grad at its view of `out`.  None for a fit of
        no step (after the batch check, before anything is rebound). """
        solver = self.solver
        nums = solver._constraint_numbers(loss_terms)
        eq_term = 'equation' in loss_terms                # reference :448: the equation term is optional (:382-389)
        fused_constraints = [e for e in (self._constraint_plan(n) for n in nums) if e is not None]
        fused_nums = tuple(n for n in nums if self._constraint_plan(n) is not None)
        nums = [n for n in nums if self._constraint_plan(n) is None]     # the rest is added by autograd
        dist = _dist()
        world = dist.get_world_size() if dist is not None else 1
        rank = dist.get_rank() if dist is not None else 0
        local_n, point_offset = shard_batch(batch_size, world, rank)
        if local_n <= 0:
            raise ValueError('batch_size %d is smaller than the number of ranks %d' % (batch_size, world))
        # weight of a point's criterion value in the loss: 1 / (global batch) — the mean of model_torch.py:448 —, or 1 for
        # criteria with reduction='sum'
        inv_n = 1.0 if self._sum_reduction() else 1.0 / float(batch_size)
        total = solver.model.total
        if niters <= 0:
            return None
        # every parameter's .grad must be the view of `out` (a previous zero_grad may have dropped it)
        for p, o in self.entries:
            if p.grad is None or p.grad.data_ptr() != self.out.data_ptr() + 4 * o:
                p.grad = self.out[o:o + p.numel()].view(p.shape)
        # parameters that came to life after the engine was built (a V() first met inside a constraint that does not
        # lower) own their .grad: the kernel never overwrites it, so it has to be cleared every step like the
        # reference does (model_torch.py:428)
        entry_ids = {id(p) for p, _ in self.entries}
        stray_params = [p for p in solver.model.parameters() if id(p) not in entry_ids]
        cols_key, cols = sampler_columns(sampler, total)
        return dict(eq_term=eq_term, cols_key=cols_key, cols=cols, local_n=local_n, inv_n=inv_n,
                    point_offset=point_offset, dist=dist, fused_constraints=fused_constraints, fused_nums=fused_nums,
                    nums=nums, stray_params=stray_params, batch_size=batch_size, total=total, criterion=criterion)

    def _fit_stepwise(self, niters, batch_size, sampler, loss_terms, criterion, opt, opt_ready):
        """ One launch of the step kernel per optimizer step, with the constraint launches, autograd's constraints and
        torch's optimizer (or the Adam in the step kernel's tail); captured in CUDA graphs where possible. """
        solver = self.solver
        self._adopt_optimizer()
        ev = self._eval_setup(niters, batch_size, sampler, loss_terms, criterion)
        if ev is None:
            return
        eq_term, fused_constraints, fused_nums, nums = ev['eq_term'], ev['fused_constraints'], ev['fused_nums'], ev['nums']
        dist, local_n, point_offset, inv_n, total = ev['dist'], ev['local_n'], ev['point_offset'], ev['inv_n'], ev['total']
        stray_params = ev['stray_params']

        # optimizer.step() inside the step kernel (pinn_step_adam) whenever the optimizer is the plain torch Adam this
        # engine builds and nothing has to touch the gradient between the kernel and the update
        capturable = bool(opt.param_groups and opt.param_groups[0].get('capturable', False))
        fused_adam = (os.environ.get('PYDENS_B200_FUSED_ADAM', '1') != '0' and plain_adam(opt) and capturable
                      and adam_steps_equal(opt)
                      and not fused_constraints and not nums and not stray_params and eq_term
                      and (dist is None or self.comm is not None))
        adam, adam_key = None, None
        if fused_adam:
            mask = self._bind_adam_state(opt)          # the optimizer's state tensors become views of flat buffers
            m_flat, v_flat, steps_flat, _ = self._adam_flat
            adam_key = adam_hyper(opt)
            lr, (b1, b2), eps, wd = adam_key
            adam = _native.PinnAdam(m_flat.data_ptr(), v_flat.data_ptr(), mask.data_ptr(), steps_flat.data_ptr(),
                                    steps_flat.numel(), lr, b1, b2, eps, wd, self.ring.data_ptr(), self.ring.numel())
            opt_ready = True                           # the state exists (zeros for a fresh optimizer)

        if dist is not None:
            # ranks may reach this fit seconds apart (rank 0 plotting or saving between fits): the in-kernel
            # all-reduce waits only a bounded time for its peers, so line the ranks up first
            dist.barrier()

        cols_key, cols = ev['cols_key'], ev['cols']
        solver.model.train()
        ring_ptr, ring_len = self.ring.data_ptr(), self.ring.numel()

        def one_step(points=None, full_points=None):
            if fused_adam:
                self._step_adam(points, cols, local_n, inv_n, point_offset, adam, allreduce=dist is not None)
                return
            self._evaluate(ev, points, full_points)
            opt.step()
            _native.check(self.lib.pinn_record_loss(self.plan, C.c_void_p(self.out.data_ptr()),
                                                    C.c_void_p(ring_ptr), C.c_int64(ring_len),
                                                    C.c_void_p(self.step_counter.data_ptr()), self._stream()))

        graphs_ok = (capturable or fused_adam) and not nums and os.environ.get('PYDENS_B200_NO_GRAPH') != '1'
        if cols_key is not None:
            vals = self._loop_in_kernel_sampler(niters, one_step, graphs_ok, opt_ready,
                                                ('dev', batch_size, local_n, cols_key, fused_nums, adam_key))
        else:
            vals = self._loop_host_batches(niters, batch_size, local_n, point_offset, sampler, one_step, graphs_ok,
                                           ('host', batch_size, local_n, fused_nums, adam_key), nums, dist)
        self._end_stepwise(vals, dist)

    def _evaluate(self, ev, points=None, full_points=None):
        """ The objective of a step into [grads | loss] (`out`): the equation launch (or zeros), the all-reduce, the
        fused constraint launches and the constraints autograd adds, on the step's batch (`points`: this rank's rows of
        an explicit batch, None: the in-kernel sampler's; `full_points`: the whole explicit batch, for autograd). """
        dist = ev['dist']
        if ev['eq_term']:
            self._step(points, ev['cols'], ev['local_n'], ev['inv_n'], ev['point_offset'], allreduce=dist is not None)
            if dist is not None and self.comm is None:
                dist.all_reduce(self.out)          # no peer-memory path: NCCL sums [grads | loss]
        else:
            self.out.zero_()                       # loss_terms without 'equation': the constraint terms alone
        for entry in ev['fused_constraints']:      # after the all-reduce: every rank adds the same term
            self._constraint_step(entry)
        if ev['nums']:
            # constraints that stay on autograd see the step's own batch — the WHOLE global batch, identical
            # on every rank (so that every replica adds the same gradient) and with requires_grad set, as the
            # reference hands them to the constraint (model_torch.py:436, :451-457)
            if full_points is not None:
                batch = full_points
            else:                                  # in-kernel sampler: replay the batch the kernel just drew
                batch = self.sample(ev['batch_size'], ev['cols'], point_offset=0)
            total = ev['total']
            xs = [batch[:, k:k + 1].clone().requires_grad_() for k in range(total)]
            for p in ev['stray_params']:
                p.grad = None
            closs = self.solver._constraint_loss(ev['nums'], xs, ev['criterion'])
            closs.backward()
            self.out[self.n_params] += closs.detach()

    # ------------------------------------------------------------------------------------------
    # L-BFGS: torch.optim.LBFGS.step(closure) with the update on the device (pinn_lbfgs_advance)
    def _lbfgs_bind(self, opt):
        """ The device state of `opt` -> (PinnLbfgs settings, state buffer, mask, torch-order index).  A state torch
        left in opt.state (its own steps, or a write-back that torch has stepped past since) is imported first. """
        g = opt.param_groups[0]
        m = int(g['history_size'])
        params = list(g['params'])
        pos = {id(p): o for p, o in self.entries}
        idx = torch.cat([torch.arange(pos[id(p)], pos[id(p)] + p.numel(), device=self.device) for p in params])
        mask = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
        mask[idx] = 1.0
        nbytes = self.lib.pinn_lbfgs_state_bytes(self.n_params, m)
        cur = getattr(self, '_lbfgs', None)
        if cur is None or cur['opt'] is not opt or cur['state'].numel() != nbytes or not cur['fresh'](opt):
            state = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
            cur = dict(opt=opt, state=state, m=m, idx=idx, fresh=lambda o: False)
            st = opt.state.get(params[0])
            if st and 'n_iter' in st:
                lbfgs_import(state, st, idx, self.n_params, m)
            self._lbfgs = cur
        cfg = _native.PinnLbfgs(lr=float(g['lr']), tolerance_grad=float(g['tolerance_grad']),
                                tolerance_change=float(g['tolerance_change']), max_iter=int(g['max_iter']),
                                max_eval=int(g['max_eval']), history_size=m,
                                line_search=int(g['line_search_fn'] == 'strong_wolfe'), mask=mask.data_ptr(),
                                losses_ring=self.ring.data_ptr(), ring_len=self.ring.numel(),
                                step_counter=self.step_counter.data_ptr())
        if g['line_search_fn'] not in (None, 'strong_wolfe'):
            raise RuntimeError("only 'strong_wolfe' is supported")
        return cfg, cur, mask

    def _fit_lbfgs(self, niters, batch_size, sampler, loss_terms, criterion, opt):
        """ `niters` L-BFGS steps: per evaluation of the objective (_evaluate, on the step's one batch) one
        pinn_lbfgs_advance and a read of its 4-byte status; the step counter (the in-kernel sampler's Philox step)
        moves only when the kernel finishes a step.  The device state is written back into opt.state in torch's layout
        at the end, so that torch's own opt.step(closure) can take over. """
        self._adopt_optimizer()
        ev = self._eval_setup(niters, batch_size, sampler, loss_terms, criterion)
        if ev is None:
            return
        entry_ids = {id(p) for p, _ in self.entries}
        if any(id(p) not in entry_ids for p in opt.param_groups[0]['params']):
            warnings.warn('pydens_b200: the optimizer holds parameters outside the fused network (a V() first met in a '
                          'constraint that runs on autograd): torch.optim.LBFGS runs the update, over the fused '
                          'evaluation', stacklevel=4)
            self._fit_lbfgs_torch(niters, batch_size, sampler, ev, opt)
            return
        cfg, cur, mask = self._lbfgs_bind(opt)
        dist = ev['dist']
        if dist is not None:
            dist.barrier()
        self.solver.model.train()
        status = torch.zeros(1, dtype=torch.int32, device=self.device)
        status_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        start, ring_len = self.steps_done, self.ring.numel()
        vals = np.empty(niters, dtype=np.float32)
        host = ev['cols_key'] is None
        total, off = ev['total'], ev['point_offset']
        drained = 0
        for i in _progress(niters):
            points = full = None
            if host:                                     # one host batch per step, staged once
                b = sampler.sample(batch_size)
                b = b if isinstance(b, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32))
                full = b.detach().to(self.device, torch.float32).reshape(batch_size, total).contiguous()
                if dist is not None and ev['nums']:
                    dist.broadcast(full, 0)
                points = full[off:off + ev['local_n']]
            while True:
                self._evaluate(ev, points, full if ev['nums'] else None)
                _native.check(self.lib.pinn_lbfgs_advance(
                    C.byref(cfg), C.c_int64(self.n_params), C.c_void_p(self.flat.data_ptr()),
                    C.c_void_p(self.out.data_ptr()), C.c_void_p(cur['state'].data_ptr()),
                    C.c_void_p(status.data_ptr()), self._stream()))
                status_host.copy_(status, non_blocking=True)
                torch.cuda.current_stream(self.device).synchronize()
                if int(status_host[0]) == _native.LBFGS_DONE:
                    break
            if i + 1 - drained >= ring_len:
                vals[drained:i + 1] = ring_losses(self.ring, start, drained, i + 1)
                drained = i + 1
        torch.cuda.synchronize(self.device)
        vals[drained:] = ring_losses(self.ring, start, drained, niters)
        token = lbfgs_export(cur['state'], opt, cur['idx'], self.n_params, cur['m'])
        cur['fresh'] = token
        self._end_stepwise(vals, dist)

    def _fit_lbfgs_torch(self, niters, batch_size, sampler, ev, opt):
        """ torch.optim.LBFGS.step(closure) with the fused evaluation (_evaluate) as its closure, one batch per step:
        for optimizers over parameters the device update does not hold. """
        self._lbfgs = None                               # opt.state is torch's own from here on
        dist, total, off = ev['dist'], ev['total'], ev['point_offset']
        self.solver.model.train()
        losses = []
        for _ in _progress(niters):
            points = full = None
            if ev['cols_key'] is None:
                b = sampler.sample(batch_size)
                b = b if isinstance(b, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32))
                full = b.detach().to(self.device, torch.float32).reshape(batch_size, total).contiguous()
                if dist is not None and ev['nums']:
                    dist.broadcast(full, 0)
                points = full[off:off + ev['local_n']]

            def closure():
                self._evaluate(ev, points, full if ev['nums'] else None)
                return self.out[self.n_params].clone()
            losses.append(float(opt.step(closure)))
            self.step_counter += 1                       # the next step's batch
        self.steps_done += niters
        self.solver.losses.extend(np.array(v, dtype=np.float32) for v in losses)

    def _loop_in_kernel_sampler(self, niters, one_step, graphs_ok, opt_ready, key):
        """ Points sampled in the kernel: replays of a graph of `per_graph` steps, the rest as plain launches.
        -> the losses of the `niters` steps """
        ring_len, start = self.ring.numel(), self.steps_done
        vals = np.empty(niters, dtype=np.float32)
        per_graph = int(os.environ.get('PYDENS_B200_GRAPH_STEPS', '0')) or (4 if niters >= 64 else 1)
        key += (per_graph,)
        graph = self._graphs.get(key) if graphs_ok else None
        done, drained = 0, 0
        if graphs_ok and graph is None and niters >= _GRAPH_MIN_ITERS:
            if not opt_ready:
                one_step()                        # real step 0: also materialises optimizer state
                done = 1
            try:
                torch.cuda.synchronize(self.device)

                def body():
                    for _ in range(per_graph):
                        one_step()
                # capture executes nothing, but a first launch of a freshly captured kernel sequence must not
                # be preceded by a dry run: the capture itself is side-effect free
                graph = capture_graph(self.device, body)
                self._graphs[key] = graph
            except Exception as exc:              # capture unsupported here: plain launches  # noqa: BLE001
                warnings.warn('pydens_b200: CUDA-graph capture of the step failed (%s); using plain launches' % exc)
                graph = None
                torch.cuda.synchronize(self.device)
        if graph is not None:
            for _ in range((niters - done) // per_graph):
                if done + per_graph - drained > ring_len:     # the ring is about to wrap: read it out first
                    torch.cuda.synchronize(self.device)
                    vals[drained:done] = ring_losses(self.ring, start, drained, done)
                    drained = done
                graph.replay()
                done += per_graph
        for _ in _progress(niters - done):
            if done - drained >= ring_len:
                torch.cuda.synchronize(self.device)
                vals[drained:done] = ring_losses(self.ring, start, drained, done)
                drained = done
            one_step()
            done += 1
        torch.cuda.synchronize(self.device)
        vals[drained:] = ring_losses(self.ring, start, drained, niters)
        return vals

    def _loop_host_batches(self, niters, batch_size, local_n, point_offset, host_sampler, one_step, graphs_ok, key,
                           nums, dist):
        """ Host batches through the native pipeline, one call per step (copy -> graph -> loss read once the graphs
        are captured).  -> the losses of the `niters` steps """
        total, start, stream = self.solver.model.total, self.steps_done, self._stream()
        ring_ptr, ring_len = self.ring.data_ptr(), self.ring.numel()
        # staging depth = how many steps the host may run ahead of the GPU (absorbs host jitter; matters most
        # with several ranks, where the in-kernel all-reduce makes every rank wait for the slowest host)
        n_stage = max(2, min(8, int(os.environ.get('PYDENS_B200_STAGES', '4'))))
        pkey = (local_n, n_stage)
        pipe = self._pipes.get(pkey)
        if pipe is None:
            pipe = C.c_void_p()
            _native.check(self.lib.pinn_pipe_create(self.plan, n_stage, C.c_int64(local_n), C.byref(pipe)))
            self._pipes[pkey] = pipe
        bufs = [_RawPtr(self.lib.pinn_pipe_buffer(pipe, k)) for k in range(n_stage)]
        pinned = self._pinned_batches.get((batch_size, n_stage))
        loss_host = self._pinned_losses(niters)
        loss_ptr = loss_host.data_ptr()
        key += (n_stage,)
        execs = self._graphs.get(key) if graphs_ok else None
        exec_ptrs = [g.raw_cuda_graph_exec() for g in execs] if execs else None
        keep = [None] * n_stage                    # the tensors whose memory a copy in flight still reads
        off_bytes = point_offset * total * 4
        want_graphs = graphs_ok and execs is None and niters >= _HOST_GRAPH_MIN_ITERS

        for i in _progress(niters):
            k = i % n_stage
            batch = host_sampler.sample(batch_size)
            if isinstance(batch, torch.Tensor) and batch.dtype == torch.float32 and batch.is_contiguous() \
                    and batch.device.type == 'cpu':
                src = batch                        # copied from where it lies (pinned or not)
            else:
                if pinned is None:
                    pinned = [torch.empty((batch_size, total), dtype=torch.float32).pin_memory()
                              for _ in range(n_stage)]
                    self._pinned_batches[(batch_size, n_stage)] = pinned
                _native.check(self.lib.pinn_pipe_wait(pipe, k))          # its previous copy has left the buffer
                if isinstance(batch, torch.Tensor):
                    pinned[k].copy_(batch.detach().to('cpu', torch.float32).reshape(batch_size, total))
                else:
                    pinned[k].copy_(torch.from_numpy(np.ascontiguousarray(batch, dtype=np.float32)).reshape(batch_size, total))
                src = pinned[k]
            keep[k] = src
            r = (start + i) % ring_len
            if exec_ptrs is not None:
                _native.check(self.lib.pinn_pipe_step(pipe, k, C.c_void_p(src.data_ptr() + off_bytes),
                                                      C.c_void_p(exec_ptrs[k]), C.c_void_p(ring_ptr + 4 * r),
                                                      C.c_void_p(loss_ptr + 4 * i), stream))
                continue
            _native.check(self.lib.pinn_pipe_step(pipe, k, C.c_void_p(src.data_ptr() + off_bytes), None, None, None, stream))
            full = None
            if nums:
                full = src.to(self.device, non_blocking=True)
                if dist is not None:
                    dist.broadcast(full, 0)
            one_step(bufs[k], full)
            _native.check(self.lib.pinn_pipe_finish(pipe, k, C.c_void_p(ring_ptr + 4 * r), C.c_void_p(loss_ptr + 4 * i), stream))
            # after the first (eager) step the optimizer state exists: capture the compute part of the step
            # once per staging buffer, so that every later step is ONE native call (copy -> graph -> loss read)
            if want_graphs:
                want_graphs = False
                try:
                    torch.cuda.synchronize(self.device)
                    graphs = []
                    for kk in range(n_stage):
                        graphs.append(capture_graph(self.device, lambda kk=kk: one_step(bufs[kk]),
                                                    pool=graphs[0].pool() if graphs else None))
                    self._graphs[key] = graphs
                    exec_ptrs = [g.raw_cuda_graph_exec() for g in graphs]
                except Exception as exc:        # capture unsupported here: keep plain launches  # noqa: BLE001
                    warnings.warn('pydens_b200: CUDA-graph capture of the step failed (%s); using plain launches' % exc)
                    exec_ptrs = None
                    torch.cuda.synchronize(self.device)
        torch.cuda.synchronize(self.device)
        return loss_host[:niters].numpy().copy()

    def _end_stepwise(self, vals, dist):
        """ The end of a stepwise fit of len(vals) steps: drop graphs that hold NCCL collectives, check that every
        rank reached the in-kernel all-reduce, log the losses. """
        self.steps_done += len(vals)
        if dist is not None and self.comm is None:
            # NCCL fallback: the cached graphs hold captured NCCL collectives, and NCCL's communicator teardown
            # (dist.destroy_process_group) waits for every such graph to be destroyed first — do not keep them
            self._graphs = {}
        if self.comm is not None:
            aborted = C.c_int(0)
            _native.check(self.lib.pinn_comm_status(self.comm, C.byref(aborted), 1))
            if aborted.value:
                raise RuntimeError('pydens_b200: a rank did not reach the in-kernel all-reduce within the time limit '
                                   '(PINN_COMM_TIMEOUT_S); the gradients of this fit were poisoned with NaN')
        self.solver.losses.extend(np.array(v, dtype=np.float32) for v in vals)


def _lbfgs_views(state, n_params, m):
    """ (header, fp64 arrays by name, vector slot accessor) of an L-BFGS state buffer (a uint8 device tensor) """
    lay = _native.lbfgs_layout(n_params, m)
    f64 = {k: state[o:o + 8 * c].view(torch.float64) for k, (o, c) in lay['f64'].items()}
    nv = lay['nv']
    vec = state[lay['vectors']:lay['total']].view(torch.float32)
    return lay, f64, (lambda k: vec[k * nv:(k + 1) * nv])


def lbfgs_import(state, st, idx, n_params, m):
    """ torch.optim.LBFGS's state (`st`, the dict on its first parameter; vectors in the optimizer's parameter order)
    into a zeroed device state: d, prev_flat_grad, the history pairs (oldest in slot 0) and their Gram entries, t,
    H_diag, n_iter, func_evals, prev_loss. """
    lay, f64, vec = _lbfgs_views(state, n_params, m)
    S = lay['S']
    hdr = _native.PinnLbfgsState()
    hdr.n_iter, hdr.func_evals = int(st.get('n_iter', 0)), int(st.get('func_evals', 0))
    hdr.t = float(st['t']) if st.get('t') is not None else 0.0
    hdr.H_diag = float(st['H_diag']) if st.get('H_diag') is not None else 1.0
    hdr.prev_loss = float(st['prev_loss']) if st.get('prev_loss') is not None else 0.0

    def put(k, v):
        if v is not None:
            vec(k)[idx] = v.detach().reshape(-1).to(torch.float32)
    put(_native.LBFGS_D, st.get('d'))
    put(_native.LBFGS_PG, st.get('prev_flat_grad'))
    dirs, stps = list(st.get('old_dirs') or []), list(st.get('old_stps') or [])
    k = len(dirs)
    for i in range(k):
        put(_native.LBFGS_RING + i, stps[i])
        put(_native.LBFGS_RING + S + i, dirs[i])
    if k:
        s_ = torch.stack([vec(_native.LBFGS_RING + i) for i in range(k)]).double()
        y_ = torch.stack([vec(_native.LBFGS_RING + S + i) for i in range(k)]).double()
        sy = f64['sy'].view(S, S)
        yy = f64['yy'].view(S, S)
        sy[:k, :k] = s_ @ y_.T
        yy[:k, :k] = y_ @ y_.T
    hdr.ring_count, hdr.ring_head = k, 0
    state[:C.sizeof(hdr)].copy_(torch.frombuffer(bytearray(bytes(hdr)), dtype=torch.uint8))


def lbfgs_export(state, opt, idx, n_params, m):
    """ The device state into opt.state in torch.optim.LBFGS's layout (vectors gathered in the optimizer's parameter
    order).  -> a predicate telling whether opt.state still holds exactly this write-back (torch has not stepped). """
    lay, f64, vec = _lbfgs_views(state, n_params, m)
    S = lay['S']
    hdr = _native.PinnLbfgsState.from_buffer_copy(bytes(state[:C.sizeof(_native.PinnLbfgsState)].cpu().numpy()))
    p0 = opt.param_groups[0]['params'][0]
    st = opt.state[p0]
    st['n_iter'], st['func_evals'] = int(hdr.n_iter), int(hdr.func_evals)
    if hdr.n_iter == 0:
        return lambda o: o.state.get(p0) is st and st.get('n_iter') == 0
    k, head = int(hdr.ring_count), int(hdr.ring_head)
    slots = [(head + i) % S for i in range(k)]
    sy = f64['sy'].view(S, S)
    st['d'] = vec(_native.LBFGS_D)[idx].clone()
    st['t'] = float(hdr.t)
    st['old_stps'] = [vec(_native.LBFGS_RING + p)[idx].clone() for p in slots]
    st['old_dirs'] = [vec(_native.LBFGS_RING + S + p)[idx].clone() for p in slots]
    st['ro'] = [(1.0 / sy[p, p]).float() for p in slots]
    st['H_diag'] = torch.tensor(float(hdr.H_diag), dtype=torch.float32, device=state.device)
    st['prev_flat_grad'] = vec(_native.LBFGS_PG)[idx].clone()
    st['prev_loss'] = float(hdr.prev_loss)
    al = f64['al'][:k].float()
    st['al'] = [al[i] for i in range(k)] + [None] * (int(opt.param_groups[0]['history_size']) - k)
    d = st['d']
    n_iter = st['n_iter']
    return lambda o: o.state.get(p0) is st and st.get('d') is d and st.get('n_iter') == n_iter


class _RawPtr:
    """ A device pointer with the one method `_step` needs from a tensor. """
    def __init__(self, ptr):
        self.ptr = int(ptr)

    def data_ptr(self):
        return self.ptr
