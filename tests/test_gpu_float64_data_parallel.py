"""The data-parallel training step against float64: the gradient mean, the L2 fold and the Adam update on every rank,
eager and captured.

Every other float64 check runs one process on one GPU.  What a data-parallel step adds on top of it -- the all-reduce
of the flat gradient buffer, the 1 / world factor folded into the Adam kernel (``grad_scale`` in eager mode,
``_hyper_dev[4]`` in a captured step), the L2 term the kernel adds after the mean, each rank's shard of the batch
and the captured step with the all-reduce inside the graph -- is checked here on the real Trainer, started once per
rank under ``torch.distributed.run`` (this file is also that worker; see ``_worker``).  Each rank builds the Trainer
with seed 1234, takes rank 0's variables (``broadcast_variables``), trains two steps on its own
``run.synthetic_batch`` shard and writes, after steps 0, 1 and 2, SHA-256 digests of its flat parameter and moment
buffers, its loss and the decisions it took (below); rank 0 also writes its variables and Adam slots.  The schedule halves lr after the first step (decay_after = 0, decay_interval = 1), so a
captured step has its hyper-parameter vector rewritten while world > 1.

Nothing of the product is instrumented to see what Adam was given.  Adam's first moment after step 1 is
m1 = (1 - b1) g1 to one fp32 rounding, with (1 - b1) formed in fp32 (0.100000024), and after step 2
g2 = (m2 - b1 m1) / (1 - b1).  So the effective gradient g_eff = mean_r g_r + l2 w of each step is read back from the
moments (to 1.5e-7 of the gradient Adam received, measured) and compared with float64: the objective's oracle
(tests/test_gpu_float64_objective.py; the supervised loss of tests/test_gpu_float64_network.py for the fine-tune) on
each rank's shard at the previous step's variables, averaged over the ranks.  The oracle's loss carries the
regulariser, so the mean carries l2 w once.  Each variable is scored by max(rel L2, max / max |ref|), weights and
biases separately.

The float64 side follows the decisions of the data-parallel step itself: each worker records, per step, the
leaky-ReLU sides and the level-loss calls' flows and mask bits with the objective file's recorders, and the oracle of
rank r's shard follows rank r's record (the mask bits are checked against float64_refs.masks_f32 there).  Following
another run's decisions is not enough: two 3xTF32 evaluations of C-kitti at the same variables and batch differed
by up to 1.3e-3 in a weight gradient (flow5_up4, deconv4), because a pre-activation or a mask test within rounding
of its threshold can fall either way.  The single-GPU product gradient on the same shards, scored against the same
float64 mean, is printed as a yardstick: it shows that spread.

Per case and step the file also checks:
  * replicas: the flat parameters and both moments are bit-identical on every rank, and the per-rank losses differ
    (the shards do);
  * moment consistency: v1 = (1 - b2) g1^2 and v2 = b2 v1 + (1 - b2) g2^2 with g from the first moments, in units of
    2^-24 |v| (both moments saw the same gradient, scale and L2 term);
  * the update rule: p_i = p_(i-1) - lr_i sqrt(1 - b2^i) / (1 - b1^i) m_i / (sqrt(v_i) + eps) in float64 from the
    stored fp32 values (b1, b2, eps as fp32 values, as the kernel reads them), in units of 2^-24 (|p_i| + |update|):
    lr, the step counter and eps, also after the captured step's lr rewrite;
  * frozen networks (CSS-bench): their variables do not move and they have no moments.

Transports: with two or more GPUs the ranks talk NCCL, one GPU each, as ``[run] gpu_list`` and bench.py train.
With fewer the NCCL cases skip, and the "one-gpu" cases run two ranks over gloo on cuda:0: everything above the
transport -- the factor, the L2 fold, the shards, the replicas, the Adam kernel -- in eager mode (gloo cannot be
captured).  test_run_command_matches_float64 runs ``python -m unflow_b200.run`` itself with ``gpu_list = 0,1`` and
reads the effective gradients from its checkpoints, which holds run.py's own batch split and shard choice.  That
command cannot record its decisions, so its float64 side follows a single-GPU run's and its bound
(TAU_GRAD_SPREAD) is 3x the spread above.

Measured on an H100 SXM 80 GB (HBM3) at a 700 W power limit with one GPU (worst score of g_eff per family over
steps 1 and 2 and two runs, the single-GPU yardstick's, the worst moment and update errors in units of 2^-24):

  case                              weights   biases    yardstick   moments   update
  C-kitti one-gpu eager             2.8e-5    6.2e-5    7.4e-4      5.8       3.3
  CSS-ft-train_all one-gpu eager    1.7e-3    5.0e-3    5.6e-3      5.6       3.0

Replicas were bit-identical at every step.  The fine-tune differentiates a train_all stack's image_warp, whose
floor() and |warp - im1| the float64 side does not follow (the network file's TAU_GRAD_WARP family).  Bounds: C-kitti
and CSS-bench keep the objective file's TAU_GRAD (6.2e-4, 10x the C-kitti measurement: CSS-bench's bias gradients
reached 2.1e-4 there); TAU_GRAD_FT 1.5e-2, TAU_MOMENT 18 and TAU_UPDATE 10 are 3x the worst measured.  The NCCL
cases, the bench's dp shape and the run.py command need two or more GPUs and have not been measured: in particular
bit-identity after an NCCL all-reduce is expected (reduce-scatter, then all-gather of the reduced chunks) but not
measured.

Negative controls (test_bound_catches_a_data_parallel_error), two-rank C-kitti eager, each patched into the workers
only; measured over gloo on one GPU:
  grad_scale = 1 (the sum, not the mean)            g_eff 1.03 (1655x TAU_GRAD)
  every rank trains on rank 0's shard               g_eff 1.02 (1641x TAU_GRAD)
  l2 w added on each rank before the all-reduce     g_eff 9.0e-2 (145x TAU_GRAD), the weights only
  no broadcast_variables, seeds 1234 + rank         replicas differ after steps 0, 1 and 2
With one GPU the file takes 3 to 4 minutes: 20-45 s per two-rank worker launch, most of it start-up, and 5-26 s of
float64 per case.
"""
import argparse
import hashlib
import os
import shutil
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:        # the worker runs as a script
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

import float64_refs as R  # noqa: E402
import test_gpu_float64_network as N  # noqa: E402
from test_gpu_float64_objective import _record_loss_side, assert_case, run_float64, run_product  # noqa: E402
from test_gpu_launch import _processes_mentioning  # noqa: E402
from test_gpu_variant_step_launches import CSS_BENCH_PARAMS, KITTI_FT_PARAMS, KITTI_PARAMS  # noqa: E402

pytestmark = pytest.mark.gpu

TAU_GRAD = 6.2e-4           # g_eff against float64 (see the docstring)
TAU_GRAD_FT = 1.5e-2        # the train_all fine-tune: gradients that cross image_warp's floor and |warp - im1|
# the run.py command cannot record its decisions: the float64 side follows a single-GPU run's, so g_eff carries the
# run-to-run spread of the product at one point (two 3xTF32 evaluations of C-kitti differed by up to 1.3e-3)
TAU_GRAD_SPREAD = 4e-3
TAU_MOMENT = 18.0           # units of 2^-24 |v|
TAU_UPDATE = 10.0           # units of 2^-24 (|p| + |update|)
F32 = 2.0 ** -24
TIMEOUT = 900

# id -> (loss parameters, per-rank batch, H, W, supervised)
CASES = {
    "C-kitti": (KITTI_PARAMS, 2, 320, 1152, False),
    "CSS-bench": (CSS_BENCH_PARAMS, 1, 384, 1280, False),
    "CSS-ft-train_all": (KITTI_FT_PARAMS, 2, 320, 768, True),
    "C-kitti-all": (KITTI_PARAMS, 1, 320, 1152, False),
}

# run id -> (case, mode, transport).  "nccl": one GPU per rank; "one-gpu": two ranks over gloo on cuda:0.
RUNS = {
    "C-kitti-eager": ("C-kitti", "eager", "nccl"),
    "C-kitti-graph": ("C-kitti", "graph", "nccl"),
    "CSS-bench-graph": ("CSS-bench", "graph", "nccl"),
    "CSS-ft-train_all-eager": ("CSS-ft-train_all", "eager", "nccl"),
    "CSS-ft-train_all-graph": ("CSS-ft-train_all", "graph", "nccl"),
    "C-kitti-all-eager": ("C-kitti-all", "eager", "nccl"),
    "C-kitti-one-gpu-eager": ("C-kitti", "eager", "one-gpu"),
    "CSS-ft-train_all-one-gpu-eager": ("CSS-ft-train_all", "eager", "one-gpu"),
}


def schedule(params):
    """The case's loss parameters with lr at step 1 and lr / 2 at step 2."""
    p = {k: v for k, v in params.items() if not k.startswith('manual_decay')}
    lr = params['manual_decay_lrs'][0] if 'manual_decay_lrs' in params else params['learning_rate']
    return dict(p, learning_rate=lr, decay_after=0, decay_interval=1)


def _gpus():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def world_of(cid, transport):
    if transport == "one-gpu":
        return 2
    return min(_gpus(), 8) if cid == "C-kitti-all" else 2


def _skip_reason(cid, transport):
    n = _gpus()
    if transport == "nccl" and n < 2:
        return "needs at least 2 visible GPUs for NCCL, this machine shows %d" % n
    if cid == "C-kitti-all" and n < 4:
        return "the bench's dp shape needs at least 4 visible GPUs, this machine shows %d" % n
    return None


# ---- the worker: one rank of the data-parallel step -----------------------------------------------------------------
CONTROLS = {
    "sum": "grad_scale = 1: the all-reduced sum instead of the mean",
    "rank0-shard": "every rank trains on rank 0's shard",
    "l2-before-reduce": "each rank adds l2 w before the all-reduce (the kernel adds it again)",
    "no-broadcast": "no broadcast_variables, rank-dependent initial seeds",
}


def _patch_control(control, Trainer):
    """Apply a negative control to the product, inside this worker process only."""
    real = Trainer.reduce_gradients
    if control == "sum":
        Trainer.reduce_gradients = lambda self: (real(self), 1.0)[1]
    elif control == "l2-before-reduce":
        def reduce_gradients(self):
            self.flat_grad.add_(self.l2_gradient())
            return real(self)
        Trainer.reduce_gradients = reduce_gradients


def _to(obj, device):
    """``obj`` (nested lists, tuples, dicts, namespaces of tensors) with every tensor copied to ``device``."""
    if torch.is_tensor(obj):
        return obj.detach().to(device, copy=True)
    if isinstance(obj, (list, tuple)):
        return type(obj)(_to(o, device) for o in obj)
    if isinstance(obj, dict):
        return {k: _to(v, device) for k, v in obj.items()}
    if isinstance(obj, SimpleNamespace):
        return SimpleNamespace(**_to(vars(obj), device))
    return obj


def _pack(mask):
    return (tuple(mask.shape), torch.from_numpy(np.packbits(mask.cpu().numpy().reshape(-1))))


def _unpack(packed):
    shape, bits = packed
    n = int(np.prod(shape))
    return torch.from_numpy(np.unpackbits(bits.numpy(), count=n).astype(bool)).view(shape).cuda()


def _record_decisions(m, Trainer, supervised, augment=False):
    """The recorders of the objective file (leaky-ReLU sides; the level-loss calls' flows, masks and splat maps;
    under ``augment`` the augmented images and mask) on the product, emptied at the start of every loss evaluation:
    after a step they hold that step's decisions.  In a captured step they are graph memory, which every replay
    rewrites."""
    sides = R.record_kink_sides(m)
    rec = None if supervised else _record_loss_side(m, augment)
    real = Trainer.loss

    def loss(self, *batch):
        for v in sides.values():
            del v[:]
        if rec is not None:
            del rec.levels[:]
        return real(self, *batch)
    m.setattr(Trainer, "loss", loss)
    return sides, rec


def _snapshot(tr, full):
    """SHA-256 digests of the flat parameter and moment buffers; with ``full`` also the variables and Adam slots
    (TF layout)."""
    out = dict(digest=[hashlib.sha256(t.detach().cpu().numpy().tobytes()).hexdigest()
                       for t in (tr.flat_param, tr.adam_m, tr.adam_v)])
    if full:
        out.update(vars=tr.variables.to_tf_dict(),
                   slots={k: (torch.from_numpy(m), torch.from_numpy(v)) for k, (m, v) in tr.adam_slots().items()})
    return out


def _worker(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", required=True)
    ap.add_argument("--mode", choices=("eager", "graph"), required=True)
    ap.add_argument("--transport", choices=("nccl", "one-gpu"), required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--control", choices=[""] + list(CONTROLS), default="")
    args = ap.parse_args(argv)
    import torch.distributed as dist
    from unflow_b200 import run, synthetic
    from unflow_b200.e2eflow.core import flownet
    from unflow_b200.e2eflow.core.train import Trainer
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    device = torch.device("cuda", 0 if args.transport == "one-gpu" else int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(device)
    if args.transport == "nccl":
        dist.init_process_group("nccl", device_id=device)
    else:
        dist.init_process_group("gloo")
    flownet.set_conv_precision("3xtf32")
    params, B, H, W, supervised = CASES[args.case]
    params = schedule(params)
    _patch_control(args.control, Trainer)
    seed = 1234 + rank if args.control == "no-broadcast" else 1234
    tr = Trainer(params, synthetic.KITTI_NORMALIZATION, device, seed=seed, supervised=supervised)
    if args.control != "no-broadcast":
        tr.broadcast_variables(0)
    shard = 0 if args.control == "rank0-shard" else rank
    steps = [dict(_snapshot(tr, rank == 0), loss=None, seed=None)]
    with pytest.MonkeyPatch.context() as m:
        sides, rec = _record_decisions(m, Trainer, supervised)
        for i in (1, 2):
            batch = run.synthetic_batch(B, H, W, i, shard, device, supervised=supervised)
            if args.mode == "graph" and tr._graph is None:
                tr.capture(*batch)
            loss = tr.step(*batch)
            torch.cuda.synchronize()
            steps.append(dict(_snapshot(tr, rank == 0), loss=float(loss), seed=1234 + 7919 * i + shard,
                              sides={k: [_pack(t) for t in v] for k, v in sides.items()}, rec=_to(rec, "cpu")))
    layout = dict(names=tr.trainable_names, offsets=tr._offsets, shapes=[tuple(p.shape) for p in tr.trainable])
    torch.save(dict(steps=steps, layout=layout, world=world), os.path.join(args.out, "rank%d.pt" % rank))
    torch.cuda.synchronize()
    dist.barrier()
    sys.stdout.flush()
    sys.stderr.flush()
    if args.mode == "graph" and args.transport == "nccl":
        os._exit(0)     # ncclCommDestroy hangs after the communicator was used inside a graph (run.py does the same)
    dist.destroy_process_group()
    return 0


def _launch(tmp_path, rid, control=""):
    """Run ``rid`` under torch.distributed.run: ([rank results], world)."""
    cid, mode, transport = RUNS[rid]
    world = world_of(cid, transport)
    out = tmp_path / ("%s%s" % (rid, "-" + control if control else ""))
    out.mkdir()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(world),
           os.path.abspath(__file__), "--case", cid, "--mode", mode, "--transport", transport, "--out", str(out)]
    if control:
        cmd += ["--control", control]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=TIMEOUT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    assert not _processes_mentioning(str(out)), "a worker outlived its launcher"
    results = [torch.load(str(out / ("rank%d.pt" % k)), weights_only=False) for k in range(world)]
    shutil.rmtree(out)
    return results, world


# ---- the float64 side -----------------------------------------------------------------------------------------------
def _product_layout(name, t):
    return t.permute(3, 2, 0, 1) if name.endswith('/weights') else t


def _cases(cid):
    return _case_tuples(*CASES[cid])


def _case_tuples(params, B, H, W, supervised, augment=False):
    ncase = (params['flownet'], params.get('train_all'), False, False, B, H, W, "supervised", "flat", 1)
    return params, supervised, ncase, (params, B, H, W, augment)


def shard_reference(monkeypatch, cid, tfv, batch, sides, rec):
    """{name: float64 gradient} (L2 term included, the product's layout) of the case's objective on one shard at the
    variables ``tfv``, following the decisions ``sides`` / ``rec`` the data-parallel step recorded on that shard."""
    return float64_objective(monkeypatch, CASES[cid], tfv, batch, sides, rec)[1]


def float64_objective(monkeypatch, case, tfv, batch, sides, rec, augment=False):
    """(float64 loss or None for the supervised loss, {name: float64 gradient}) of ``case`` = (loss parameters, B,
    H, W, supervised) on ``batch`` at the variables ``tfv``, following the recorded decisions ``sides`` / ``rec``
    (with ``augment``, the recorded augmented images and mask)."""
    params, supervised, ncase, ocase = _case_tuples(*case, augment=augment)
    rec = _to(rec, "cuda")
    loss = None
    with monkeypatch.context() as m:
        used, cat = R.follow_kink_sides(m, sides)
        if supervised:
            _, ref = N.run_oracle(m, ncase, tfv, [batch])
        else:
            out, ref, log = run_float64(m, ocase, tfv, batch, rec)
            assert len(log) == len(rec.levels), "level-loss calls the oracle did not make"
            assert_case(params, {}, log, [])     # the recorded mask bits are the right ones
            loss = out["loss"]
    assert all(used[k] == cat[k].shape[0] for k in cat), "activations the oracle did not consume"
    return loss, ref


def single_gpu_run(monkeypatch, cid, tfv, batch):
    """The single-GPU product on one shard: its gradient (plus the L2 term) and the decisions it took."""
    params, supervised, ncase, ocase = _cases(cid)
    with monkeypatch.context() as m:
        sides = R.record_kink_sides(m)
        if supervised:
            return N.run_product(ncase, tfv, [batch])[1], sides, None
        rec = _record_loss_side(m, False)
        return run_product(m, ocase, tfv, batch, "3xtf32", rec)[1], sides, rec


def _score(got, ref):
    rows = {"weights": [], "biases": []}
    assert set(got) == set(ref), sorted(set(got) ^ set(ref))
    for name, r in ref.items():
        l2, mx = R.errors(got[name], r)
        rows["weights" if name.endswith('/weights') else "biases"].append((max(l2, mx), l2, mx, name))
    return rows


def _moments_before(states, i, name):
    """(m, v) of ``name`` after step i - 1, float64: zeros before the first step (no slot recorded)."""
    prev = states[i - 1].get("slots") or {}
    if name not in prev:
        return 0.0, 0.0
    return tuple(t.double() for t in prev[name])


def effective_gradients(states, steps=(1, 2)):
    """{step: {name: g_eff}} in the product's layout, float64, from the first moments of ``steps`` and of the
    step before each: g_i = (m_i - b1 m_(i-1)) / (1 - b1)."""
    b1 = float(torch.tensor(0.9, dtype=torch.float32))
    c1 = float(torch.tensor(1.0) - torch.tensor(0.9))       # 1 - b1 as the kernel forms it: 0.100000024
    out = {i: {} for i in steps}
    for i in steps:
        for name, (m, _) in states[i]["slots"].items():
            m_prev = _moments_before(states, i, name)[0]
            out[i][name] = _product_layout(name, (m.double() - b1 * m_prev) / c1).cuda()
    return out


def moment_errors(states, steps=(1, 2)):
    """Worst |v_i - v_i(g_i)| over ``steps`` and elements, in units of 2^-24 |v| (2^-126 at least)."""
    b1, b2 = (float(torch.tensor(b, dtype=torch.float32)) for b in (0.9, 0.999))
    c1, c2 = (float(torch.tensor(1.0) - torch.tensor(b)) for b in (0.9, 0.999))
    worst = 0.0
    for i in steps:
        for name, (m, v) in states[i]["slots"].items():
            m_prev, v_prev = _moments_before(states, i, name)
            m, v = m.double(), v.double()
            g = (m - b1 * m_prev) / c1
            want = b2 * v_prev + c2 * g * g
            err = (v - want).abs() / (F32 * want.abs().clamp_min(2.0 ** -126))
            worst = max(worst, float(err.max()))
    return worst


def update_errors(states, params, steps=(1, 2)):
    """Worst |p_i - p_i(Adam)| over ``steps`` and elements, in units of 2^-24 (|p_i| + |update|)."""
    from unflow_b200.e2eflow.core.train import learning_rate_at
    b1, b2, eps = (float(torch.tensor(b, dtype=torch.float32)) for b in (0.9, 0.999, 1e-8))
    worst = 0.0
    for i in steps:
        lr_t = learning_rate_at(i - 1, params) * (1 - b2 ** i) ** 0.5 / (1 - b1 ** i)
        for name, (m, v) in states[i]["slots"].items():
            p0, p1 = states[i - 1]["vars"][name].double(), states[i]["vars"][name].double()
            upd = lr_t * m.double() / (v.double().sqrt() + eps)
            err = (p1 - (p0 - upd)).abs() / (F32 * (p1.abs() + upd.abs()).clamp_min(2.0 ** -126))
            worst = max(worst, float(err.max()))
    return worst


def _mean(gs):
    return {k: sum(g[k].double() for g in gs) / len(gs) for k in gs[0]}


def score_steps(monkeypatch, cid, states, shards, decisions):
    """g_eff of steps 1 and 2 (from ``states``' moments) against the float64 mean over the shards, each at the
    decisions ``decisions(i, r)`` returns for step i's shard r (None: the single-GPU yardstick's own), and the
    yardstick against the same; the moment and update errors."""
    geff = effective_gradients(states)
    rows, yard = {}, {}
    for i in (1, 2):
        tfv = states[i - 1]["vars"]
        refs, singles = [], []
        for r, b in enumerate(shards[i]):
            grads, sides, rec = single_gpu_run(monkeypatch, cid, tfv, b)
            singles.append(grads)
            recorded = decisions(i, r)
            refs.append(shard_reference(monkeypatch, cid, tfv, b, *(recorded or (sides, rec))))
        ref = _mean(refs)
        rows[i] = _score(geff[i], ref)
        yard[i] = _score(_mean(singles), ref)
    return rows, yard, moment_errors(states), update_errors(states, schedule(CASES[cid][0]))


def _recorded(results):
    return lambda i, r: ({k: [_unpack(t) for t in v] for k, v in results[r]["steps"][i]["sides"].items()},
                         results[r]["steps"][i]["rec"])


def grad_bound(cid):
    params = CASES[cid][0]
    return TAU_GRAD_FT if params.get('train_all') and len(params['flownet']) > 1 else TAU_GRAD


def report(title, rows, yard, moments, update, seconds):
    lines = ["%s (%.1f s)" % (title, seconds)]
    for i in (1, 2):
        for fam in ("weights", "biases"):
            w, y = max(rows[i][fam]), max(yard[i][fam])
            lines.append("  step %d %-8s g_eff %.3e (rel L2 %.3e, max %.3e, %s); single-GPU mean %.3e"
                         % (i, fam, w[0], max(r[1] for r in rows[i][fam]), max(r[2] for r in rows[i][fam]), w[3],
                            y[0]))
    lines.append("  moments %.2f x 2^-24, update %.2f x 2^-24" % (moments, update))
    return "\n".join(lines)


def worst_grad(rows):
    return max(r for i in (1, 2) for fam in ("weights", "biases") for r in rows[i][fam])


def replica_diffs(results):
    """The steps (0, 1, 2) after which some rank's flat parameters or moments differ from rank 0's in a bit."""
    return [i for i in range(3) if any(r["steps"][i]["digest"] != results[0]["steps"][i]["digest"]
                                       for r in results[1:])]


def check_run(monkeypatch, cid, results, world):
    """Every check of one worker run; returns the report."""
    t0 = time.time()
    params, B, H, W, supervised = CASES[cid]
    from unflow_b200 import run
    diffs = replica_diffs(results)
    assert not diffs, "replicas differ after steps %s" % diffs
    for i in (1, 2):
        losses = [r["steps"][i]["loss"] for r in results]
        assert len(set(losses)) == world, "per-rank losses of step %d: %s" % (i, losses)
        assert len({r["steps"][i]["seed"] for r in results}) == world
    states = results[0]["steps"]
    trainable = N._trainable(params['flownet'], params.get('train_all'), list(states[0]["vars"]))
    assert set(states[1]["slots"]) == trainable, "moments of variables that are not trained"
    for name in set(states[0]["vars"]) - trainable:     # frozen networks
        for i in (1, 2):
            assert torch.equal(states[i]["vars"][name], states[0]["vars"][name]), name
    shards = {i: [run.synthetic_batch(B, H, W, i, r, "cuda", supervised=supervised) for r in range(world)]
              for i in (1, 2)}
    rows, yard, moments, update = score_steps(monkeypatch, cid, results[0]["steps"], shards, _recorded(results))
    return rows, yard, moments, update, time.time() - t0


def assert_scores(cid, rows, moments, update, tau=None):
    tau = tau or grad_bound(cid)
    for i in (1, 2):
        for fam in ("weights", "biases"):
            assert max(rows[i][fam])[0] <= tau, "step %d %s: %s" % (i, fam, max(rows[i][fam]))
    assert moments <= TAU_MOMENT, moments
    assert update <= TAU_UPDATE, update


@pytest.mark.parametrize("rid", list(RUNS))
def test_data_parallel_step_matches_float64(monkeypatch, tmp_path, rid):
    cid, mode, transport = RUNS[rid]
    reason = _skip_reason(cid, transport)
    if reason:
        pytest.skip(reason)
    t0 = time.time()
    results, world = _launch(tmp_path, rid)
    rows, yard, moments, update, dt = check_run(monkeypatch, cid, results, world)
    print("\n" + report("%s, world %d, worker %.1f s" % (rid, world, time.time() - t0 - dt), rows, yard, moments,
                        update, dt))
    print("  losses per rank, step 1: %s" % [r["steps"][1]["loss"] for r in results])
    assert_scores(cid, rows, moments, update)


# ---- negative controls ----------------------------------------------------------------------------------------------
def _control_run():
    return "C-kitti-eager" if _gpus() >= 2 else "C-kitti-one-gpu-eager"


@pytest.mark.parametrize("control", list(CONTROLS))
def test_bound_catches_a_data_parallel_error(monkeypatch, tmp_path, control):
    """Two-rank C-kitti eager with one error patched into the worker: the replica check must fail at every step
    (no-broadcast), or g_eff must exceed TAU_GRAD by 30x (the others)."""
    rid = _control_run()
    results, world = _launch(tmp_path, rid, control)
    diffs = replica_diffs(results)
    if control == "no-broadcast":
        print("\n%s: replicas differ after steps %s" % (control, diffs))
        assert diffs == [0, 1, 2]
        return
    assert not diffs, diffs
    rows, yard, moments, update, dt = check_run_unchecked(monkeypatch, "C-kitti", results, world)
    w = worst_grad(rows)
    print("\n" + report("%s, %s" % (rid, control), rows, yard, moments, update, dt))
    print("%s: worst g_eff %.3e = %.0f x TAU_GRAD (%s)" % (control, w[0], w[0] / TAU_GRAD, w[3]))
    assert w[0] > 30 * TAU_GRAD


def check_run_unchecked(monkeypatch, cid, results, world):
    """check_run's scores without its replica and shard assertions (a control breaks those on purpose)."""
    t0 = time.time()
    params, B, H, W, supervised = CASES[cid]
    from unflow_b200 import run
    shards = {i: [run.synthetic_batch(B, H, W, i, r, "cuda", supervised=supervised) for r in range(world)]
              for i in (1, 2)}
    rows, yard, moments, update = score_steps(monkeypatch, cid, results[0]["steps"], shards, _recorded(results))
    return rows, yard, moments, update, time.time() - t0


# ---- the real command -----------------------------------------------------------------------------------------------
CFG = """
[dirs]
log = {d}/log
checkpoints = {d}/log/checkpoints
data = {d}/nodata
[run]
batch_size = 4
gpu_list = 0,1
dataset = kitti
development = False
conv_precision = 3xtf32
[train]
save_interval = 1
display_interval = 1
flownet = C
pyramid_loss = True
border_mask = True
ternary_weight = 1.0
smooth_2nd_weight = 3.0
[train_kitti]
height = 320
width = 1152
num_iters = 2
learning_rate = 1.0e-5
decay_after = 0
decay_interval = 1
fb_weight = 0.2
mask_occlusion = fb
occ_weight = 12.4
"""


@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_run_command_matches_float64(monkeypatch, tmp_path, mode):
    """``python -m unflow_b200.run`` on gpu_list = 0,1 (batch_size 4, so 2 per rank): g_eff of steps 1 and 2 from
    the Adam slots of model.ckpt-1.pt and model.ckpt-2.pt against float64 over the shards synthetic_batch gives
    ranks 0 and 1 at each step."""
    if _gpus() < 2:
        pytest.skip("needs at least 2 visible GPUs, this machine shows %d" % _gpus())
    from unflow_b200 import run
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    ini = tmp_path / "config.ini"
    ini.write_text(CFG.format(d=tmp_path))
    cmd = [sys.executable, "-m", "unflow_b200.run", "--ex", "dp", "--config", str(ini), "--synthetic",
           "--no-augment", "--max-iters", "2"] + (["--graph"] if mode == "graph" else [])
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=TIMEOUT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    assert not _processes_mentioning(str(ini))
    cfg = run.config_dict(str(ini))
    params = dict(cfg["train"], **cfg["train_kitti"])
    assert schedule(dict(KITTI_PARAMS)) == {k: params[k] for k in schedule(dict(KITTI_PARAMS))}
    states = [dict(vars=FlowNetVariables('C', False, seed=1234).to_tf_dict(), slots={})]
    for i in (1, 2):
        ck = torch.load(str(tmp_path / "log" / "checkpoints" / "dp" / ("model.ckpt-%d.pt" % i)))
        states.append(dict(vars=ck["variables"], slots=ck["adam_slots"]))
    shards = {i: [run.synthetic_batch(2, 320, 1152, i, k, "cuda") for k in range(2)] for i in (1, 2)}
    rows, yard, moments, update = score_steps(monkeypatch, "C-kitti", states, shards, lambda i, r: None)
    print("\n" + report("run.py gpu_list = 0,1, %s" % mode, rows, yard, moments, update, 0.0))
    assert_scores("C-kitti", rows, moments, update, TAU_GRAD_SPREAD)


if __name__ == "__main__":
    sys.exit(_worker(sys.argv[1:]))
