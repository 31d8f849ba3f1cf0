/*
 * pinn_b200.h — C ABI of the H100-native PINN fit-step engine.
 *
 * This is the drop-in boundary for the ONE hot path of analysiscenter/pydens that this
 * repository replaces: the body of the training loop of `Solver.fit`
 * (reference: pydens/model_torch.py:426-464).  The reference has no FFI layer of its own
 * (it is pure Python on PyTorch autograd), so every entry point below cites the reference
 * lines whose work it takes over.  The Python host side (pydens_b200/solver.py) binds this
 * library with ctypes; see INTEGRATION.md for the binding a pydens maintainer would add.
 *
 * Conventions
 *   - All `float*` / `void*` data pointers are DEVICE pointers owned by the caller
 *     (PyTorch tensors), borrowed for the duration of the call, 16-byte aligned.
 *   - All calls are stream-ordered on `stream` (a cudaStream_t passed as void*), perform
 *     no allocation and no host synchronisation, and are CUDA-graph capturable
 *     (pinn_plan_create / pinn_plan_destroy excepted: they query the device and set kernel
 *     attributes and must not be called during capture).  The plan travels to the kernels as a
 *     __grid_constant__ parameter: there is no device-side plan object to keep alive.
 *   - Return value: 0 on success, negative PINN_E_* on failure; pinn_last_error() gives a
 *     thread-local human readable message.
 *   - A plan is immutable after creation and may be used from several streams.
 *
 * No torch types appear in this interface.
 */
#ifndef PINN_B200_H
#define PINN_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PINN_ABI_VERSION   11

#define PINN_MAX_LAYERS    16   /* linear layers                                   */
#define PINN_MAX_DIMS       8   /* ndims + nparams (columns of the point matrix)   */
#define PINN_MAX_DIRS       6   /* first-order derivative directions (NF)          */
#define PINN_MAX_VARS       4   /* scalar V() variables used inside the equation   */
#define PINN_MAX_PROG     192   /* instructions per expression program             */
#define PINN_MAX_SLOTS     96   /* scratch slots of an expression program          */

/* error codes */
#define PINN_OK             0
#define PINN_E_INVALID     -1   /* malformed spec / argument                       */
#define PINN_E_UNSUPPORTED -2   /* valid request outside what the kernels cover    */
#define PINN_E_CUDA        -3   /* CUDA runtime error (message has the detail)     */
#define PINN_E_ALIGN       -4   /* pointer not 16-byte aligned                     */
#define PINN_E_WORKSPACE   -5   /* workspace too small                             */

/* activation ids (reference: batchflow Block `activation=` names used by
 * pydens/model_torch.py:158-168; 'Tanh' README.md:41, 'Sigmoid' model_torch.py:159) */
#define PINN_ACT_NONE       0
#define PINN_ACT_TANH       1
#define PINN_ACT_SIGMOID    2
#define PINN_ACT_SIN        3   /* sin z (batchflow-style `Sin` callable, model_torch.py:150-151) */
#define PINN_ACT_SOFTPLUS   4   /* nn.Softplus() with default beta / threshold     */
#define PINN_ACT_SILU       5   /* nn.SiLU()                                       */
#define PINN_ACT_GELU       6   /* nn.GELU() (erf form)                            */

/* expression-program opcodes: a tiny register machine evaluated once per collocation
 * point.  Programs are produced on the host by tracing the user's `equation` /
 * `initial_condition` callables (reference: the opaque Python callables invoked at
 * pydens/model_torch.py:448 and :127) and differentiating them symbolically. */
enum PinnOp {
    PINN_OP_CONST = 0,  /* dst = imm                                   */
    PINN_OP_COORD = 1,  /* dst = x[a]            (column a of the point) */
    PINN_OP_VAR   = 2,  /* dst = V[a]            (a-th equation variable) */
    PINN_OP_ADD   = 3,  /* dst = s[a] + s[b]     */
    PINN_OP_SUB   = 4,
    PINN_OP_MUL   = 5,
    PINN_OP_DIV   = 6,
    PINN_OP_NEG   = 7,  /* dst = -s[a]           */
    PINN_OP_MULI  = 8,  /* dst = s[a] * imm      */
    PINN_OP_ADDI  = 9,  /* dst = s[a] + imm      */
    PINN_OP_SIN   = 10,
    PINN_OP_COS   = 11,
    PINN_OP_EXP   = 12,
    PINN_OP_LOG   = 13,
    PINN_OP_SQRT  = 14,
    PINN_OP_TANH  = 15,
    PINN_OP_POWI  = 16, /* dst = s[a] ** (int)imm */
    PINN_OP_POW   = 17, /* dst = powf(s[a], s[b]) */
    PINN_OP_ABS   = 18,
    PINN_OP_SIGN  = 19,
    PINN_OP_SIGMOID = 20,
    PINN_OP_RECIP = 21, /* dst = 1 / s[a]        */
    PINN_OP_TAN   = 22,
    PINN_OP_COUNT_
};

typedef struct PinnInstr {
    uint8_t op, dst, a, b;
    float   imm;
} PinnInstr;

/* sampler column kinds (reference: default `torch.rand` columns model_torch.py:431 and
 * batchflow NumpySampler 'uniform'/'normal' used at README.md:82, tutorial cell `NS('u', ...)`) */
#define PINN_COL_UNIFORM    0   /* a + (b - a) * U[0,1)   */
#define PINN_COL_NORMAL     1   /* a + b * N(0,1)          */
#define PINN_COL_CONST      2   /* a                       */
#define PINN_COL_MIXTURE    3   /* one of n_comp simple columns, drawn per point (batchflow `s1 | s2`) */
#define PINN_COL_TNORMAL    4   /* a + b * N(0,1) conditioned on comp_a[0] <= value <= comp_b[0]: batchflow
                                   `NumpySampler('n', ...).truncate(high, low)` by rejection — up to 16 re-draws on
                                   further Philox blocks, then the value is clamped into the interval           */
#define PINN_MAX_MIX        4

/* A mixture column picks component i with probability cum_w[i] - cum_w[i-1] (cum_w[n_comp-1] == 1) and then
 * samples (comp_kind[i], comp_a[i], comp_b[i]) like a simple column.  Columns that carry the same `group`
 * share the draw of the component — `(a1 & a2) | (b1 & b2)` picks the whole row from one side. */
typedef struct PinnColumn {
    int32_t kind;
    float   a, b;
    int32_t group;                       /* 0 .. PINN_MAX_DIMS-1 (mixture columns only)                 */
    int32_t n_comp;                      /* 2 .. PINN_MAX_MIX                                           */
    float   cum_w[PINN_MAX_MIX];
    int32_t comp_kind[PINN_MAX_MIX];     /* PINN_COL_UNIFORM / NORMAL / CONST                           */
    float   comp_a[PINN_MAX_MIX], comp_b[PINN_MAX_MIX];
} PinnColumn;

/*
 * Everything that defines one `Solver`: network, ansatz, derivative jet set, residual.
 *
 * Network (reference ConvBlockModel.forward model_torch.py:170-172, layouts 'fa…f'):
 *   n_layers linear layers, widths[0] = ndims + nparams, widths[n_layers] = k, the number of outputs: 1, or 2..4 for
 *   coupled systems (derivative order <= 2, nf <= 4; see Programs), which run on the thread kernel, or on the tile
 *   kernel's 128-wide class when their 65-128-wide hidden layers do not fit the thread kernel's shared memory;
 *   act[l] is the activation applied AFTER linear layer l (0-based); act[n_layers-1] must
 *   be PINN_ACT_NONE.  skip_src[l] = s >= 0 adds the output of layer s (after ITS activation and skip)
 *   to the activated output of layer l (residual connections 'R … +').
 * Flat parameter buffer (fp32): for layer l the weight matrix [widths[l+1] x widths[l]]
 *   row-major (== torch nn.Linear.weight) at w_off[l] and the bias at b_off[l]; the scalar
 *   log_scale (model_torch.py:50) at log_scale_off; equation variables (V token,
 *   model_torch.py:180-188) at var_off[i].  n_params = number of floats in the buffer,
 *   rounded up by the caller to a multiple of 4.  The gradient buffer uses the same layout.
 *
 * Ansatz (reference TorchModel.anzatc model_torch.py:107-128):
 *   has_bc: u = N * prod_i g_i(x_i) + bc_value over the first ndims_spatial columns,
 *           g_i(x) = (x - lo_i)(hi_i - x) / (hi_i - lo_i)^2;
 *   has_ic: u = (sigmoid((t - t0) / exp(log_scale)) - 0.5) * u + ic(x_spatial),
 *           t = column ndims-1, t0 = dom_lo[ndims-1], ic given by ic_prog.
 *
 * Jet set (what the nested D() calls of the equation need, model_torch.py:174-178):
 *   nf first-order directions; direction d is the vector dir_vec[d][0..ndims+nparams) in point-column
 *   space (dir_col[d] = k >= 0 when it is the unit vector of column k, else -1); the first ns (<= nf)
 *   of them additionally carry the second directional derivative along the same vector.  Mixed
 *   derivatives d2u/dx_i dx_j are obtained by polarisation from the direction e_i + e_j:
 *   u_ij = (u_vv - u_ii - u_jj) / 2.  Channel order of every jet: [value, D_dir0.., D^2_dir0 ..].
 *
 * Programs: scratch slots 0..C-1 (C = 1 + nf + ns) are preloaded with the jet of u before
 *   eq_prog runs.  eq_out[0] is the slot of the residual r, eq_out[1+c] the slot of
 *   dr/d(jet channel c), eq_out[1+C+i] the slot of dr/dV_i.  ic_prog runs before u is
 *   assembled; ic_out[c] is the slot holding channel c of the jet of ic.  When the initial condition
 *   uses variables (ic_has_vars; e.g. README.md:112-118 `V('init', ...)`), ic_out[C*(1+i) + c] is the
 *   slot of d(ic jet channel c)/dV_i and those slots lie above every slot eq_prog writes.
 *   Networks of k = 2..4 outputs: slots j*C + c are preloaded with channel c of component j; eq_out[0] is still the
 *   residual; the partials dr/d(channel c of component j) form one contiguous block, slot eq_out[1] + j*C + c, so that
 *   eq_out[1 + c] = eq_out[1] + c; eq_out[1 + C + i] is still dr/dV_i.  ic_out is unchanged (one initial condition,
 *   shared by every component like the boundary value, boundary factor and time gate).
 */
typedef struct PinnSpec {
    int32_t  abi_version;
    int32_t  n_layers;
    int32_t  widths[PINN_MAX_LAYERS + 1];
    int32_t  act[PINN_MAX_LAYERS];
    int32_t  skip_src[PINN_MAX_LAYERS];   /* -1, or the earlier layer whose (activated) output is added to this
                                             layer's activated output: layouts 'faR fa fa+ f' (model_torch.py:142-156) */
    int32_t  w_off[PINN_MAX_LAYERS];
    int32_t  b_off[PINN_MAX_LAYERS];
    int32_t  n_params;
    int32_t  log_scale_off;
    int32_t  n_vars;
    int32_t  var_off[PINN_MAX_VARS];

    int32_t  ndims, nparams;
    int32_t  has_bc, has_ic;
    float    bc_value;
    float    dom_lo[PINN_MAX_DIMS], dom_hi[PINN_MAX_DIMS];

    int32_t  nf, ns;                      /* first-order directions, and how many of them (the first ns) also carry a second
                                             derivative.  nf <= 4: any ns <= nf.  nf = 5, 6 (full Hessians in 3-D, Laplacians
                                             in 5 / 6 dimensions): ns = nf only — a direction the equation differentiates once
                                             still carries its second-order channel, with a zero entry in eq_out's partials */
    int32_t  dir_col[PINN_MAX_DIRS];
    float    dir_vec[PINN_MAX_DIRS][PINN_MAX_DIMS];

    int32_t   n_eq;
    PinnInstr eq_prog[PINN_MAX_PROG];
    int32_t   eq_out[1 + 1 + 2 * PINN_MAX_DIRS + PINN_MAX_VARS];
    int32_t   n_ic;
    PinnInstr ic_prog[PINN_MAX_PROG];
    int32_t   ic_out[(1 + 2 * PINN_MAX_DIRS) * (1 + PINN_MAX_VARS)];
    int32_t   ic_has_vars;
    int32_t   n_slots;          /* scratch slots either program may touch */
    int32_t   order;            /* 0 (or 2): derivatives up to order 2, channels = value, nf firsts, ns seconds (above).
                                   3 or 4 (D nested three / four times, model_torch.py:174-178: u_xxx of KdV, u_xxxx of beam
                                   equations): EVERY direction carries its Taylor jet up to this order — channel
                                   1 + d*order + (k-1) holds the k-th derivative along direction d, channels = 1 + nf*order;
                                   ns is ignored (0); nf <= 4 (axes, and diagonals e_i +- e_j that carry mixed derivatives by
                                   polarisation) */
} PinnSpec;

typedef struct PinnPlan PinnPlan;

/* Thread-local message of the last failing call. */
const char* pinn_last_error(void);

/* ABI version of the loaded library (== PINN_ABI_VERSION of the header it was built from). */
int pinn_abi_version(void);

/* Validate `spec`, pick the kernel variant for its jet set and widths, upload the device
 * copy.  Host-side, done once per Solver — the counterpart of Solver.__init__'s model
 * construction (model_torch.py:312-325); NOT on the hot path. */
int pinn_plan_create(const PinnSpec* spec, int device, PinnPlan** out);
int pinn_plan_destroy(PinnPlan* plan);

/* Bytes of device workspace pinn_step / pinn_forward need for up to `n_points` points per
 * call.  (Cross-CTA partial sums, the grid ticket, and — for networks whose activations do
 * not fit shared memory — the activation spill area.) */
size_t pinn_workspace_bytes(const PinnPlan* plan, int64_t n_points);

/* Number of floats of the `grads_and_loss` buffer: n_params (multiple of 4) + 4. */
int pinn_out_floats(const PinnPlan* plan);

/*
 * ONE fit step minus the optimizer: replaces model_torch.py:430-460, i.e. sampling (:430-436),
 * concat (:437), model forward + ansatz (:438), the D()-built residual (:448), MSE (:448) and
 * loss.backward() (:460).
 *
 *   params          [n_params] flat fp32 parameters.
 *   points          [n_points, ndims+nparams] row-major fp32, or NULL to sample in-kernel.
 *   cols            (points == NULL) host pointer to ndims+nparams column descriptors; NULL
 *                   means U[0,1) on every column (reference default, model_torch.py:431).
 *   seed            Philox key.
 *   step_counter    device pointer to a uint64 step number (Philox counter word; advanced
 *                   by pinn_record_loss) or NULL to use `step_value`.
 *   point_offset    global index of this call's first point (rank shard offset), so that the
 *                   sampled stream does not depend on how the batch is sharded.
 *   n_points        points processed by THIS call.
 *   inv_global_n    1 / (global batch size): the MSE mean of model_torch.py:448 is taken over
 *                   the global batch, so per-rank outputs simply add up.
 *   grads_and_loss  [n_params + 4] overwritten: d(loss)/d(params) in params layout, then
 *                   [n_params] = this call's share of the loss (sum r^2 * inv_global_n).
 *   residual_out    optional [n_points] per-point residual (debug / parity), or NULL.
 */
int pinn_step(const PinnPlan* plan,
              const float* params,
              const float* points,
              const PinnColumn* cols,
              uint64_t seed,
              const uint64_t* step_counter,
              uint64_t step_value,
              uint64_t point_offset,
              int64_t n_points,
              float inv_global_n,
              float* grads_and_loss,
              float* residual_out,
              void* workspace, size_t workspace_bytes,
              void* stream);

/*
 * Data-parallel runs: the all-reduce of [grads | loss] fused into the tail of the step kernel, over
 * NVLink peer memory — no NCCL call, no extra launch.  (The reference has no multi-device path; this
 * is the native form of "one all-reduce of the tiny gradient buffer per step".)
 *
 *   pinn_comm_create   allocates this rank's exchange buffer (cudaMalloc inside the library so that it
 *                      can be shared through CUDA IPC) and returns its 64-byte IPC handle;
 *   pinn_comm_connect  maps the buffers of all ranks of the SAME node from their handles (gathered by
 *                      the caller, e.g. with torch.distributed.all_gather_object), rank-ordered;
 *   pinn_step_allreduce  == pinn_step, except that `grads_and_loss` receives the SUM over all ranks:
 *                      the last CTA stores the rank's vector into its slot of every rank's buffer
 *                      (peer stores), publishes an arrival flag (release, system scope), waits for the
 *                      flags of all ranks and sums the slots in rank order, so every rank holds
 *                      bit-identical results.  All ranks must issue the same sequence of calls.  If a
 *                      peer does not arrive within PINN_COMM_TIMEOUT_S (default 60) seconds the outputs are set to NaN instead of
 *                      hanging; pinn_comm_status reports (and clears) that condition.
 */
#define PINN_COMM_HANDLE_BYTES 64
#define PINN_COMM_MAX_RANKS     8
typedef struct PinnComm PinnComm;
int pinn_comm_create(const PinnPlan* plan, int rank, int world, PinnComm** comm,
                     unsigned char handle_out[PINN_COMM_HANDLE_BYTES]);
int pinn_comm_connect(PinnComm* comm, const unsigned char* handles /* world x 64 bytes, rank order */);
int pinn_comm_destroy(PinnComm* comm);
int pinn_step_allreduce(const PinnPlan* plan, const PinnComm* comm,
                        const float* params, const float* points, const PinnColumn* cols,
                        uint64_t seed, const uint64_t* step_counter, uint64_t step_value,
                        uint64_t point_offset, int64_t n_points, float inv_global_n,
                        float* grads_and_loss, float* residual_out,
                        void* workspace, size_t workspace_bytes, void* stream);

/* Health of the peer all-reduce: *aborted != 0 after a peer failed to arrive within the time limit (the step's
 * outputs were poisoned with NaN and the flag is sticky).  Host-synchronous (one 4-byte D2H); call it after a fit,
 * not per step.  `reset` != 0 clears the flag.  PINN_COMM_TIMEOUT_S in the environment sets the limit (default 60 s). */
int pinn_comm_status(PinnComm* comm, int* aborted, int reset);

/*
 * Host-batch pipeline: the per-step HOST work of the reference loop when the points come from a host sampler —
 * `sampler.sample(batch_size)` -> tensors on the device (model_torch.py:433-437) and `losses.append(loss.cpu())`
 * (:464) — as ONE native call per step.  The pipe owns `n_stage` device staging buffers ([local_n, total] fp32),
 * a copy stream and a read-back stream:
 *
 *   pinn_pipe_step(pipe, slot, host_points, graph_exec, ring_src, loss_dst, stream)
 *       1. copy stream: wait until the compute stream no longer reads staging buffer `slot`, then
 *          cudaMemcpyAsync(host_points -> buffer[slot])            (host_points: local_n*total floats, pinned);
 *       2. `stream` (the compute stream) waits for that copy;
 *       3. cudaGraphLaunch(graph_exec, stream) — the captured compute part of the step
 *          (pinn_step on buffer[slot] + optimizer + pinn_record_loss); skipped when graph_exec is NULL
 *          (the caller launches the step itself and then calls pinn_pipe_finish);
 *       4. read-back stream: after the step, cudaMemcpyAsync(loss_dst <- ring_src, 4 bytes) (loss_dst pinned).
 *   pinn_pipe_finish   steps 4 of the above for a caller-launched step (graph_exec == NULL).
 *   pinn_pipe_wait     host-blocks until the H2D copy last issued for `slot` has completed (the caller may then
 *                      overwrite the pinned source it handed in);   pinn_pipe_sync drains both side streams.
 * Nothing here allocates per step; the calls are NOT capturable (they are the part of the step that stays outside
 * the CUDA graph).
 */
typedef struct PinnPipe PinnPipe;
int pinn_pipe_create(const PinnPlan* plan, int n_stage, int64_t local_n, PinnPipe** out);
int pinn_pipe_destroy(PinnPipe* pipe);
float* pinn_pipe_buffer(PinnPipe* pipe, int slot);
int pinn_pipe_step(PinnPipe* pipe, int slot, const float* host_points, void* graph_exec,
                   const float* ring_src, float* loss_dst, void* stream);
int pinn_pipe_finish(PinnPipe* pipe, int slot, const float* ring_src, float* loss_dst, void* stream);
int pinn_pipe_wait(PinnPipe* pipe, int slot);
int pinn_pipe_sync(PinnPipe* pipe);

/*
 * ONE fit step INCLUDING optimizer.step() and the loss log: pinn_step / pinn_step_allreduce (model_torch.py:430-460)
 * with torch.optim.Adam's update (:461) and `losses.append` (:464) executed in the tail of the same kernel by the CTA
 * that holds the reduced gradient — one launch per step instead of four (step, two fused-Adam kernels, loss record).
 * `comm` may be NULL (single GPU) or a connected communicator (every rank applies the bit-identical update).
 * `params` is updated IN PLACE; `grads_and_loss` still receives [grads | loss] of the step.  The Adam state belongs to
 * the caller (on the Python side: views that torch's optimizer object shares, so `optimizer.step()` and this call are
 * interchangeable from one step to the next).  t = 1 + max(step_tensors); every step tensor += 1;
 * losses_ring[*step_counter % ring_len] = loss (skipped when losses_ring is NULL); ++*step_counter.
 * Capturable in a CUDA graph (the step number and t live on the device).
 */
typedef struct PinnAdam {
    float* exp_avg;            /* device [n_params], in/out */
    float* exp_avg_sq;         /* device [n_params], in/out */
    const float* mask;         /* device [n_params]: 1 = trainable, 0 = frozen (left untouched) */
    float* step_tensors;       /* device [n_step_tensors] fp32 step counters of the optimizer */
    int32_t n_step_tensors;
    float lr, beta1, beta2, eps, weight_decay;
    float* losses_ring;        /* device, or NULL */
    int64_t ring_len;
} PinnAdam;
int pinn_step_adam(const PinnPlan* plan, const PinnComm* comm_or_null, float* params, const float* points,
                   const PinnColumn* cols, uint64_t seed, uint64_t* step_counter, uint64_t point_offset,
                   int64_t n_points, float inv_global_n, float* grads_and_loss, float* residual_out,
                   void* workspace, size_t workspace_bytes, const PinnAdam* adam, void* stream);

/*
 * `k_steps` WHOLE optimizer steps in one launch — the body of the reference loop including optimizer.step()
 * (model_torch.py:427-464) — for the small-batch regime where a step is launch-latency bound (README.md:36-53:
 * batch_size=100, niters=1500).  One CTA keeps the parameters, both Adam moments and the gradient in shared memory
 * between the steps.  Adam follows torch.optim.Adam (no amsgrad):  m <- lerp(m, g, 1-beta1),
 * v <- beta2 v + (1-beta2) g^2,  p <- p - lr/(1-beta1^t) * m / (sqrt(v)/sqrt(1-beta2^t) + eps),  t = opt_step0 + 1 ...
 *
 *   params, exp_avg, exp_avg_sq   [n_params] in/out;   mask [n_params]: 1 = trainable, 0 = frozen (left untouched)
 *   step_tensors                  the optimizer's per-tensor step counters (fp32 scalars laid out contiguously), += k_steps
 *   points                        [k_steps, n_points, ndims+nparams] explicit batches, or NULL (+ cols) to sample in-kernel
 *   step_counter                  device step number: Philox counter word and ring index, as in pinn_step; += k_steps
 *   losses_ring[(step) % ring_len] receives the loss of every step.
 * pinn_multi_step_max_points: largest batch the kernel takes (0: this network does not fit the kernel).
 *
 * pinn_multi_step_terms: the same with constraint terms (reference :451-457, `loss_terms=['equation', 'constraint_0']`).
 * One optimizer step is the gradient of  point_weight * sum_batch r^2  +  sum_k term_k.point_weight * sum_{its points} r_k^2,
 * and the logged loss is that sum.  point_weight is 1 / n_points for a mean criterion, 1 for reduction='sum'.
 * A term is a constraint plan (pinn_plan_create on a spec whose residual program is the constraint, evaluated on the
 * jet of u at fixed points) with the same layer table, n_params and log_scale_off as `plan`, the same ansatz, and
 * variables among the plan's.  Its jet set is either empty (nf = ns = 0: the program reads u alone, C = 1) or exactly
 * the plan's (the same nf, ns, dir_vec and order 2: it reads every channel c of the plan's jet in slot c, and its
 * eq_out holds dr/d(channel c) for all C channels, as an equation program's does) — a constraint such as u'(0) = 0
 * differentiates u at its points through the jets the kernel already carries.  Its points are read from HOST memory during the call and travel to the
 * kernel by value, with the residual program: the call allocates nothing and stays stream-ordered and capturable.
 * They do not consume sampler counters: an in-kernel batch is the one pinn_sample gives.  At most PINN_MAX_TERMS terms
 * and PINN_MAX_TERM_POINTS points in all; n_points + the term points <= pinn_multi_step_max_points.  A term plan that
 * does not match: PINN_E_INVALID.  pinn_multi_step is this call with point_weight = 1 / n_points and no terms.
 */
#define PINN_MAX_TERMS        4
#define PINN_MAX_TERM_POINTS 32
typedef struct PinnTerm {
    const PinnPlan* plan;      /* the constraint's plan */
    int32_t n_points;          /* 1 .. PINN_MAX_TERM_POINTS */
    float point_weight;        /* 1 / n_points (mean criterion) or 1 (reduction='sum') */
    const float* points;       /* HOST [n_points, ndims+nparams] row-major fp32 */
} PinnTerm;
int pinn_multi_step_max_points(const PinnPlan* plan);
int pinn_multi_step(const PinnPlan* plan, float* params, float* exp_avg, float* exp_avg_sq, const float* mask,
                    float* step_tensors, int n_step_tensors, const float* points, const PinnColumn* cols,
                    uint64_t seed, uint64_t* step_counter, int64_t n_points, int k_steps,
                    float lr, float beta1, float beta2, float eps, float weight_decay, float opt_step0,
                    float* losses_ring, int64_t ring_len, void* stream);
int pinn_multi_step_terms(const PinnPlan* plan, float* params, float* exp_avg, float* exp_avg_sq, const float* mask,
                          float* step_tensors, int n_step_tensors, const float* points, const PinnColumn* cols,
                          uint64_t seed, uint64_t* step_counter, int64_t n_points, int k_steps,
                          float lr, float beta1, float beta2, float eps, float weight_decay, float opt_step0,
                          float* losses_ring, int64_t ring_len, float point_weight, int n_terms,
                          const PinnTerm* terms, void* stream);

/*
 * ENSEMBLES of tiny-batch fits in one launch: pinn_multi_step_terms for `n_members` fits of the same plan side by side,
 * one CTA (multi-step kernel) or one cluster (cluster kernel) per member.  A PinnMember holds what differs between the
 * fits: their parameters, Adam state, mask, step tensors, step counter, loss ring, explicit batches (or NULL: sample
 * in-kernel with `cols` from the member's seed) and optimizer step count; everything else — plan, constraint terms,
 * batch size, k_steps, Adam hyper-parameters (per member: pinn_multi_step_ensemble_adam below), ring_len, point
 * weight — is shared.  Every member's result is bit-identical
 * to pinn_multi_step_terms on that member alone: the kernel and the cluster size are chosen by the same rule, and the
 * members never exchange anything.  The arguments are checked as pinn_multi_step_terms checks them, member by member;
 * n_members outside 1..PINN_MAX_MEMBERS, a null or misaligned (params: 16 bytes) member pointer: PINN_E_INVALID.
 * The member table travels to the kernel by value: the call allocates nothing and stays stream-ordered and capturable.
 */
#define PINN_MAX_MEMBERS 128
typedef struct PinnMember {
    float* params;             /* device [n_params] in/out, 16-byte aligned */
    float* exp_avg;            /* device [n_params] in/out */
    float* exp_avg_sq;         /* device [n_params] in/out */
    const float* mask;         /* device [n_params]: 1 = trainable, 0 = frozen */
    float* step_tensors;       /* device [n_step_tensors] fp32 step counters of the member's optimizer, += k_steps */
    int32_t n_step_tensors;
    float opt_step0;           /* optimizer steps the member took before this launch */
    const float* points;       /* device [k_steps, n_points, ndims+nparams], or NULL: sample in-kernel */
    uint64_t seed;
    uint64_t* step_counter;    /* device step number of the member, += k_steps */
    float* losses_ring;        /* device [ring_len] */
} PinnMember;
int pinn_multi_step_ensemble(const PinnPlan* plan, int n_members, const PinnMember* members, int64_t n_points,
                             int k_steps, float lr, float beta1, float beta2, float eps, float weight_decay,
                             int64_t ring_len, float point_weight, int n_terms, const PinnTerm* terms,
                             const PinnColumn* cols, void* stream);

/*
 * Hyper-parameter SWEEPS: pinn_multi_step_ensemble with Adam hyper-parameters of each member's own — member j steps with
 * hyper[j] (host memory, n_members rows), the way torch.optim.Adam(lr=..., betas=(beta1, beta2), eps=..., weight_decay=...)
 * would step that fit alone.  Everything else is checked and shared exactly as in pinn_multi_step_ensemble, and every
 * member's result is bit-identical to pinn_multi_step_terms on that member alone with its own row; pinn_multi_step_ensemble
 * is this call with every row equal to its shared arguments.  The rows are checked as torch.optim.Adam's constructor
 * checks them: a null `hyper`, lr or eps non-finite or < 0, beta1 or beta2 outside [0, 1), weight_decay non-finite or
 * < 0: PINN_E_INVALID, before anything launches.  The rows travel to the kernel by value with the member table.
 */
typedef struct PinnAdamHyper {
    float lr, beta1, beta2, eps, weight_decay;
} PinnAdamHyper;
int pinn_multi_step_ensemble_adam(const PinnPlan* plan, int n_members, const PinnMember* members,
                                  const PinnAdamHyper* hyper, int64_t n_points, int k_steps, int64_t ring_len,
                                  float point_weight, int n_terms, const PinnTerm* terms, const PinnColumn* cols,
                                  void* stream);

/* Forward only: u = ansatz(net(x)) for explicit points — the work of Solver.predict
 * (model_torch.py:466-487) and of the `_forward` closure handed to constraints (:451-454).
 * u_out [n_points] for a network of one output, [n_points, k] row-major for k outputs. */
int pinn_forward(const PinnPlan* plan,
                 const float* params,
                 const float* points,
                 int64_t n_points,
                 float* u_out,
                 void* workspace, size_t workspace_bytes,
                 void* stream);

/* Write the points the in-kernel sampler would produce for (seed, step, point_offset ..)
 * to points_out [n_points, ndims+nparams]: lets tests replay a sampled batch explicitly. */
int pinn_sample(const PinnPlan* plan,
                const PinnColumn* cols,
                uint64_t seed,
                const uint64_t* step_counter,
                uint64_t step_value,
                uint64_t point_offset,
                int64_t n_points,
                float* points_out,
                void* stream);

/* losses_ring[*step_counter % ring_len] = grads_and_loss[n_params]; ++*step_counter.
 * The device-side replacement for `self.losses.append(loss.detach().cpu().numpy())`
 * (model_torch.py:464), which forces a host sync every iteration in the reference. */
int pinn_record_loss(const PinnPlan* plan,
                     const float* grads_and_loss,
                     float* losses_ring, int64_t ring_len,
                     uint64_t* step_counter,
                     void* stream);

/* Introspection for tests / bench: kernel variant actually selected. */
typedef struct PinnPlanInfo {
    int32_t nf, ns, channels;
    int32_t threads_per_cta;
    int32_t ctas_per_sm;
    int32_t activations_in_smem;      /* 1: shared memory, 0: global workspace           */
    int32_t smem_bytes;
    int32_t regs_per_thread;
    int32_t sm_count;
    int32_t rows_per_point;           /* floats of per-point state kept between fwd/bwd  */
    int64_t flops_per_point;          /* algorithmic 6*C*M (SURVEY.md 8d)                */
    int32_t bytes_per_point;          /* algorithmic 4*(ndims+nparams)                   */
    int32_t tensor_core;              /* 1: the tensor-core tile kernel for wide networks runs the step (3xTF32,
                                            hidden widths <= 64),
                                         2: its 128-wide class runs it (hidden widths up to 128; networks whose
                                            weights the thread kernel cannot hold in shared memory, with 1 or
                                            2..4 outputs),
                                         0: the thread-per-point FP32 kernel                 */
    int32_t small_batch_points;       /* largest batch the cluster (point, unit)-parallel loop kernel takes through
                                         pinn_multi_step (8 CTAs x 128 points), 0: the network does not fit it         */
} PinnPlanInfo;
int pinn_plan_info(const PinnPlan* plan, PinnPlanInfo* info);

/*
 * L-BFGS ON THE DEVICE: torch.optim.LBFGS.step(closure) (torch 2.11, torch/optim/lbfgs.py) as a state machine whose
 * state lives in one device buffer.  The caller evaluates the objective (pinn_step and whatever it adds to
 * [grads | loss]) at `params`, then calls pinn_lbfgs_advance, which consumes that evaluation, writes into `params` the
 * point of the next evaluation (or the step's final point) and sets *status (device int):
 *   PINN_LBFGS_EVALUATE  evaluate again at `params` and call pinn_lbfgs_advance again (the same step goes on),
 *   PINN_LBFGS_DONE      the step is finished: losses_ring[*step_counter % ring_len] = the loss of the step's first
 *                        evaluation (what step(closure) returns; skipped when losses_ring is NULL); ++*step_counter.
 * Every branch of torch's step is restated: the first iteration's d = -g and t = min(1, 1/|g|_1) lr, the ys > 1e-10
 * memory update over a ring of history_size pairs, H_diag, the gtd > -tolerance_change break, the fixed step without
 * re-evaluation on the last inner iteration, every exit test (opt_cond at entry, max_iter, max_eval, opt_cond,
 * max|d t| <= tolerance_change, |loss - prev_loss| < tolerance_change), and _strong_wolfe with _cubic_interpolate
 * (c1 = 1e-4, c2 = 0.9, max_ls = max_eval - evaluations so far).  Only entries with mask = 1 take part in any dot
 * product, norm or update.  Dot products and scalars are fp64, vectors fp32; every reduction has a fixed order, so runs
 * are bit-reproducible.  One CTA; stream-ordered, capturable, allocates nothing.  A zeroed state buffer of
 * pinn_lbfgs_state_bytes(n_params, history_size) bytes is a fresh optimizer.  lr < 0, max_iter < 1, max_eval < 1,
 * history_size < 1, line_search not 0 / 1, a null pointer: PINN_E_INVALID.
 */
#define PINN_LBFGS_DONE          0
#define PINN_LBFGS_EVALUATE      1
typedef struct PinnLbfgs {
    double lr, tolerance_grad, tolerance_change;
    int32_t max_iter, max_eval, history_size;
    int32_t line_search;       /* 0: fixed step (line_search_fn=None), 1: 'strong_wolfe' */
    const float* mask;         /* device [n_params]: 1 = in the optimizer, 0 = frozen or padding */
    float* losses_ring;        /* device [ring_len], or NULL */
    int64_t ring_len;
    uint64_t* step_counter;    /* device step number (the in-kernel sampler's Philox step), += 1 per finished step */
} PinnLbfgs;

/*
 * The state buffer: this header, then fp64 arrays, then fp32 vectors.  With S = history_size + 1 (ring slots: the
 * pairs held plus the one the next pair is written to), nv = n_params rounded up to a multiple of 4:
 *   offset PINN_LBFGS_HEADER_BYTES:  double sy[S][S]  (sy[p][q] = s_p . y_q, physical slots), yy[S][S],
 *                                    sg[S], yg[S] (s_p . g, y_p . g of the last direction), al[S], cs[S], cy[S]
 *                                    (torch's `al`, and d = hg g + sum_i cs[i] s_i + cy[i] y_i, logical order)
 *   offset pinn_lbfgs_vector_offset(history_size), each nv floats:  0 d, 1 prev_flat_grad, 2 x (line-search base),
 *                                    3..5 line-search gradient copies, 6..6+S-1 s slots, 6+S..6+2S-1 y slots.
 * Pair i (0 = oldest) of the history sits in physical slot (ring_head + i) % S.
 */
#define PINN_LBFGS_HEADER_BYTES 512
typedef struct PinnLbfgsState {
    /* torch's state */
    int64_t n_iter, func_evals;
    double t, H_diag, prev_loss;
    int32_t ring_count, ring_head;
    /* the running step */
    int32_t phase, cur_iter, current_evals, opt_cond, g_src, action, act_arg, act_eval;
    double loss, first_loss, gtd, d_norm, gsum_g, hg;
    /* _strong_wolfe */
    int32_t ls_iter, ls_evals, max_ls, ls_done, ls_zoom, insuf, low, high, gp_ref, new_ref;
    double t_prev, f_prev, gtd_prev, f_new, gtd_new;
    double br_t[2], br_f[2], br_gtd[2];
    int32_t br_g[2];
    double ref_gmax[5];        /* max|g| of the gradients the state refers to: the evaluation, prev_flat_grad, copies */
    /* results of the last vector pass */
    double r_dot, r_max, r_l1;
} PinnLbfgsState;
size_t pinn_lbfgs_state_bytes(int64_t n_params, int history_size);
size_t pinn_lbfgs_vector_offset(int history_size);
int pinn_lbfgs_advance(const PinnLbfgs* cfg, int64_t n_params, float* params, const float* grads_and_loss,
                       void* state, int* status, void* stream);

/*
 * L-BFGS IN THE PERSISTENT CLUSTER KERNEL: `n_steps` whole L-BFGS steps of a tiny-batch fit in one launch, with no
 * launch and no host synchronisation between the evaluations of a step.  Each evaluation is the objective of
 * pinn_multi_step_terms (the batch at point_weight, plus the constraint terms) at the current parameters; cluster rank 0
 * then runs the state machine of pinn_lbfgs_advance on its shared-memory copy of the parameters, and the other CTAs of
 * the cluster copy the parameters it asks to evaluate.  A step draws its batch once, at the step number *step_counter
 * has when it begins (or reads points[s], s = 0 .. n_steps-1, [n_steps, n_points, ndims+nparams] on the device), and
 * keeps it for all of its evaluations; when the step is done the state machine logs its first loss and advances the
 * counter, exactly as pinn_lbfgs_advance does.  The state buffer has the layout of pinn_lbfgs_advance, so the two calls
 * continue each other's state.  cfg->mask, losses_ring (not NULL here) and step_counter are the fit's, cfg->lr its step
 * size.  Stream-ordered, capturable, allocates nothing.
 *   plans without the cluster kernel (PinnPlanInfo.small_batch_points == 0): PINN_E_UNSUPPORTED;
 *   a null pointer, n_steps < 1, n_points + constraint points outside 1 .. small_batch_points, settings
 *   pinn_lbfgs_advance refuses, and what pinn_multi_step_terms refuses in the terms: PINN_E_INVALID.
 * The cluster size is that of pinn_multi_step_terms for the same columns (PINN_SMALL_CLUSTER overrides).
 *
 * pinn_lbfgs_multi_ensemble: the same for n_members (1 .. PINN_MAX_MEMBERS) fits of one plan side by side, one cluster
 * each.  A PinnLbfgsMember holds what differs between them; cfg's lr, mask, losses_ring and step_counter are not read,
 * every other setting (and the terms, batch size, point weight, columns) is shared.  The members share nothing at run
 * time: each one's result is bit-identical to pinn_lbfgs_multi on it alone.
 */
typedef struct PinnLbfgsMember {
    float* params;             /* device [n_params] in/out, 16-byte aligned */
    void* state;               /* device L-BFGS state buffer (pinn_lbfgs_state_bytes) in/out */
    const float* mask;         /* device [n_params]: 1 = in the optimizer */
    const float* points;       /* device [n_steps, n_points, ndims+nparams], or NULL: sample in-kernel */
    uint64_t seed;
    uint64_t* step_counter;    /* device step number of the member, += n_steps */
    float* losses_ring;        /* device [cfg->ring_len] */
    double lr;
} PinnLbfgsMember;
int pinn_lbfgs_multi(const PinnPlan* plan, const PinnLbfgs* cfg, float* params, void* state, const float* points,
                     const PinnColumn* cols, uint64_t seed, int64_t n_points, int n_steps, float point_weight,
                     int n_terms, const PinnTerm* terms, void* stream);
int pinn_lbfgs_multi_ensemble(const PinnPlan* plan, const PinnLbfgs* cfg, int n_members, const PinnLbfgsMember* members,
                              const PinnColumn* cols, int64_t n_points, int n_steps, float point_weight, int n_terms,
                              const PinnTerm* terms, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PINN_B200_H */
