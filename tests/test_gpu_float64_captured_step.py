"""The captured training step on one GPU against float64: the step bench.py times, replay by replay.

bench.py times Trainer.capture's graph by default, and ``python -m unflow_b200.run --graph`` trains on it, but every
single-GPU float64 check runs the eager step.  A captured step runs its host code once, at capture: the tc_conv and
tc_wgrad plans and stream-K schedules, the workspace and stream-K storage pointers, the gradient-slot generations of
conv_ops, the static input buffers, the hyper-parameter vector and its device-side step counter (capture's warm-ups
run at lr = 0; it then restores the moments and resets the counter), the Philox offset of in-graph augmentation.  The
replays repeat what it decided then, while step() rewrites lr when the schedule moves and copies each batch into the
static inputs.

Each case builds the Trainer as its workload does, captures, and replays three times on three distinct
run.synthetic_batch batches.  The schedule halves lr after every step (decay_after = 0, decay_interval = 1, the
data-parallel file's schedule()), so lr is rewritten between replays.  Nothing in the graph is instrumented: the
method is tests/test_gpu_float64_data_parallel.py's.  The leaky-ReLU sides and the level-loss calls' flows, mask bits
and splat maps (and the augmented images and mask) are recorded with its _record_decisions; they are graph memory,
which every replay rewrites, so they are copied out after each replay.  The effective gradient of replay i is read
back from the first moments, g_i = (m_i - b1 m_(i-1)) / (1 - b1), and scored against the float64 objective at the
variables before the replay, following that replay's decisions.  Per replay the file checks:
  * g_eff against float64 (weights and biases, max(rel L2, max / max |ref|)), TAU_GRAD;
  * moment consistency, v_i = b2 v_(i-1) + (1 - b2) g_i^2, in units of 2^-24 |v|, TAU_MOMENT;
  * the update rule p_i = p_(i-1) - lr_i sqrt(1 - b2^i) / (1 - b1^i) m_i / (sqrt(v_i) + eps) in units of
    2^-24 (|p_i| + |update|), TAU_UPDATE: lr after each rewrite, the step counter and eps;
  * the loss the replay returned against the float64 loss, TAU_LOSS of the objective file;
  * graph_replays and the device step counter (_hyper_dev[5] = iteration + 1).
and per case: capture leaves the parameters and both moments bit-identical, the counter at iteration + 1, and the
entry points its warm-ups and its captured step call are native_entry_points.captured() of the eager step's.

The float64 side runs per sample and averages (float64_per_sample): every loss term is a Charbonnier sum over its
element count, so the batch gradient is the mean of the per-sample gradients, with the L2 term once
(test_batch_gradient_is_the_mean_of_per_sample_gradients pins that on the CPU).  Batch 4 at 384x1280 then needs the
float64 memory of one sample.

  case                      shape                   what it covers
  C-bench                   C, 4 x 384x1280         bench.run_ours' Trainer (pinned to bench.py's parameters)
  CSS-bench                 CSS, 2 x 384x1280       bench --spec CSS --batch 2: frozen C and S stay put, no moments
  C-kitti-augment-prefetch  C, 2 x 320x1152         augment=True on the device RNG, as run.py trains; replays 2 and 3
                                                    through prefetch / step_prefetched; fresh draws per replay
  C-kitti-resumed           C, 2 x 320x1152         two eager steps, then capture: replay 1 is step 3

The check found one error in the product.  The captured step's Adam formed the bias correction in fp32 on the device,
lr sqrtf(1 - powf(b2, t)) / (1 - powf(b1, t)); 1 - b2^t is 1e-3 t, so the fp32 rounding of the power (3e-8) became a
3e-6 relative error of lr_t from step 2 on, while the eager step forms lr_t in double on the host.  The update rule
measured 58.9 and 53.2 (x 2^-24) on replays 2 and 3 of C-bench, 58.1 and 53.0 on CSS-bench, against 2.8 and 3.2 on
replay 1, where t = 1 makes the power exact.  csrc/adam.cu now forms lr_t in double on the device too, as the host
does; the captured and eager steps then take the same lr_t.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, per replay (step): the worst g_eff score per family, the
moment and update errors in units of 2^-24, the loss error relative to the float64 loss:

  case                      step   weights   biases    moments   update   loss
  C-bench                   1      3.4e-5    2.7e-5    3.35      2.83     7.3e-8
                            2      2.4e-5    3.4e-5    5.85      2.65     2.5e-8
                            3      4.6e-5    3.8e-5    5.51      2.25     5.1e-8
  CSS-bench                 1      2.8e-5    3.0e-5    3.35      2.83     2.4e-7
                            2      2.8e-5    5.7e-5    5.70      2.31     1.1e-7
                            3      2.7e-5    8.5e-6    5.32      2.31     2.5e-7
  C-kitti-augment-prefetch  1      3.4e-5    5.5e-5    3.35      3.02     2.3e-8
                            2      3.8e-5    6.9e-5    5.77      3.04     1.1e-8
                            3      3.7e-5    9.6e-5    5.57      2.55     2.3e-8
  C-kitti-resumed           3      6.4e-5    4.9e-5    5.47      2.13     8.4e-8
                            4      6.4e-5    7.9e-5    5.19      2.53     1.1e-7
                            5      3.9e-5    4.1e-4    5.15      2.98     4.1e-8

These are the eager step's figures (the objective file's C-kitti 2.0e-5 / 1.9e-5, the data-parallel file's moments
5.8 and update 3.3), so the bounds that already apply to them stay: TAU_MOMENT 18 and TAU_UPDATE 10 of the
data-parallel file, TAU_LOSS 2.1e-5 of the objective file.  The one outlier is C-kitti-resumed's step-5 flow6/biases
(two elements on the 5x18 level): 4.1e-4 in the run above and 6.6e-4 in another, which moves with the float atomics'
order as the objective file's worst bias gradient does, and is over the data-parallel file's TAU_GRAD (6.2e-4).  So
TAU_GRAD here is 2.0e-3, 3x that worst measurement.  The GPU tests of the file take 136 s (C-bench 33 s, CSS-bench
27 s, the 320x1152 cases 19-20 s, the controls 5-14 s); peak memory is 6.0 GB (C-bench; float64 one sample at a
time).

Negative controls (test_bound_catches_a_captured_step_error), each patched into the product only, measured as above:
  the static inputs are not refreshed on replay 2 (C-kitti-resumed)        g_eff 2.6 (1316x TAU_GRAD)
  capture leaves the step counter where its warm-ups left it               update 7.0e6 x 2^-24 (702669x TAU_UPDATE)
    (C-kitti-augment-prefetch, replay 1 at t = 4 instead of 1)
  a resumed capture does not restore the moments (C-kitti-resumed)         moments 1.1e7 x 2^-24 (633396x TAU_MOMENT),
                                                                           g_eff 2.6 (1302x TAU_GRAD)
"""
import gc
import time
from types import SimpleNamespace

import pytest
import torch

import float64_refs as R
import native_entry_points as EP
import test_gpu_float64_data_parallel as DP
from test_gpu_float64_objective import TAU_LOSS
from test_gpu_variant_step_launches import CSS_BENCH_PARAMS, KITTI_PARAMS

TAU_GRAD = 2.0e-3               # g_eff against float64: 3x the worst measured (see the docstring)
TAU_MOMENT = DP.TAU_MOMENT      # units of 2^-24 |v|
TAU_UPDATE = DP.TAU_UPDATE      # units of 2^-24 (|p| + |update|)
REPLAYS = 3

# bench.run_ours: dict(synth.KITTI_PARAMS, learning_rate=1.0e-5, flownet=args.spec)
C_BENCH_PARAMS = dict(KITTI_PARAMS)

# id -> (loss parameters, B, H, W, augment, eager steps before capture, how replays 2.. get their batch,
#        entry points of capture's warm-ups and captured step)
CASES = {
    "C-bench": (C_BENCH_PARAMS, 4, 384, 1280, False, 0, "step", EP.CAPTURED_STEP_CALLS),
    "CSS-bench": (CSS_BENCH_PARAMS, 2, 384, 1280, False, 0, "step",
                  EP.captured(EP.VARIANT_STEP_CALLS["CSS-bench"])),
    "C-kitti-augment-prefetch": (KITTI_PARAMS, 2, 320, 1152, True, 0, "prefetch",
                                 EP.captured(EP.AUGMENT_STEP_CALLS)),
    "C-kitti-resumed": (KITTI_PARAMS, 2, 320, 1152, False, 2, "step", EP.CAPTURED_STEP_CALLS),
}


# ---- the float64 side per sample --------------------------------------------------------------------------------
def sample_sides(sides, B, b):
    """The leaky-ReLU sides of sample b: rows b, B + b, 2B + b, ... of each scope's calls.  The product's calls over
    B or 2B images (both images, both directions) are blocks of B, which the oracle's calls over one sample take
    one row of each, in the same order."""
    out = {}
    for k, v in sides.items():
        cat = torch.cat(v, 0)
        assert cat.shape[0] % B == 0, (k, tuple(cat.shape))
        out[k] = [cat[b::B]]
    return out


def sample_of(obj, B, b):
    """``obj`` (nested lists, tuples, dicts, namespaces of [B, ...] tensors) with every tensor cut to sample b."""
    if torch.is_tensor(obj):
        assert obj.shape[0] == B, tuple(obj.shape)
        return obj[b:b + 1]
    if isinstance(obj, (list, tuple)):
        return type(obj)(sample_of(o, B, b) for o in obj)
    if isinstance(obj, dict):
        return {k: sample_of(v, B, b) for k, v in obj.items()}
    if isinstance(obj, SimpleNamespace):
        return SimpleNamespace(**sample_of(vars(obj), B, b))
    return obj


def float64_per_sample(monkeypatch, params, B, H, W, augment, tfv, batch, sides, rec):
    """(float64 loss, {name: float64 gradient}) of the batch as the mean over its samples, each following its own
    recorded decisions."""
    losses, grads = [], []
    for b in range(B):
        loss, g = DP.float64_objective(monkeypatch, (params, 1, H, W, False), tfv, [t[b:b + 1] for t in batch],
                                       sample_sides(sides, B, b), sample_of(rec, B, b), augment=augment)
        losses.append(loss)
        grads.append(g)
        torch.cuda.empty_cache()
    return float(sum(losses) / B), DP._mean(grads)


# ---- the product ------------------------------------------------------------------------------------------------
class _Names:
    """Stands in for the library handle and records the entry points called through it."""

    def __init__(self, real):
        self._real = real
        self.calls = set()

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name.startswith("unflow_"):
            self.calls.add(name)
        return fn


def _record_step_calls(m, native, Trainer):
    """The entry points every capture-mode step (capture's warm-ups and the captured step) calls, through a
    library handle that only records their names."""
    names = _Names(native.lib())
    real = Trainer._step_impl

    def step_impl(self, *batch):
        m.setattr(native, "_lib", names)
        try:
            return real(self, *batch)
        finally:
            m.setattr(native, "_lib", names._real)
    m.setattr(Trainer, "_step_impl", step_impl)
    return names


def _stale_inputs(m, Trainer):
    """step() does not copy the batch into the static inputs on replay 2: the graph trains on replay 1's batch."""
    real = Trainer.step

    def step(self, *batch, lr=None):
        if self._graph is not None and self.graph_replays == 1:
            batch = tuple(self._static)         # a copy onto itself: the static inputs keep replay 1's batch
        return real(self, *batch, lr=lr)
    m.setattr(Trainer, "step", step)


def _stale_counter(m, Trainer):
    """capture() leaves the device step counter where its lr = 0 warm-ups left it."""
    real = Trainer._set_hyper

    def set_hyper(self, lr, step):
        if self._graph is None and lr != 0.0:       # capture's reset after the warm-ups
            torch.cuda.synchronize(self.device)
            step = float(self._hyper_dev[5])
        return real(self, lr, step)
    m.setattr(Trainer, "_set_hyper", set_hyper)


def _unrestored_moments(m, Trainer):
    """capture() leaves the moments its lr = 0 warm-ups fed instead of restoring the resumed run's."""
    real_impl, real_set = Trainer._step_impl, Trainer._set_hyper

    def step_impl(self, *batch):
        out = real_impl(self, *batch)
        if not torch.cuda.is_current_stream_capturing():
            self._warm_moments = (self.adam_m.clone(), self.adam_v.clone())
        return out

    def set_hyper(self, lr, step):
        if self._graph is None and lr != 0.0:       # capture() has just put the moments back
            self.adam_m.copy_(self._warm_moments[0])
            self.adam_v.copy_(self._warm_moments[1])
        return real_set(self, lr, step)
    m.setattr(Trainer, "_step_impl", step_impl)
    m.setattr(Trainer, "_set_hyper", set_hyper)


# control -> (patch, case, replays, the families that must catch it)
CONTROLS = {
    "static inputs not refreshed": (_stale_inputs, "C-kitti-resumed", 2, ("g_eff",)),
    "step counter not reset": (_stale_counter, "C-kitti-augment-prefetch", 1, ("update",)),
    "moments not restored": (_unrestored_moments, "C-kitti-resumed", 1, ("moments", "g_eff")),
}


def run_captured(monkeypatch, cid, control=None, replays=REPLAYS):
    """Case ``cid`` on the product: {step: state} with the variables and Adam slots before the first eager step,
    after every eager step and after every replay (each replay's state with its loss, counters and the decisions
    it recorded), the state capture left, the counter after capture, and the entry points the capture called."""
    from unflow_b200 import _native, run, synthetic
    from unflow_b200.e2eflow.core import augment as aug
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core.train import Trainer
    params, B, H, W, augment, eager, feed, _ = CASES[cid]
    dev = torch.device("cuda", 0)
    batch = lambda i, where=dev: run.synthetic_batch(B, H, W, i, 0, where)
    with monkeypatch.context() as m:
        m.setattr(aug, "_device_rng", aug._device_rng)     # (the Trainer turns it on for augment)
        prev = conv_ops.get_mode()
        conv_ops.set_mode("3xtf32")
        try:
            if control is not None:
                CONTROLS[control][0](m, Trainer)
            sides, rec = DP._record_decisions(m, Trainer, False, augment)
            tr = Trainer(DP.schedule(params), synthetic.KITTI_NORMALIZATION, dev, seed=1234, augment=augment)
            if augment:
                aug.seed(4321)          # as run.py seeds rank 0
            states = {0: DP._snapshot(tr, True)}
            for i in range(1, eager + 1):
                tr.step(*batch(i))
                torch.cuda.synchronize()
                states[i] = DP._snapshot(tr, True)
            first = eager + 1
            names = _record_step_calls(m, _native, Trainer)
            tr.capture(*batch(first))
            torch.cuda.synchronize()
            after_capture = DP._snapshot(tr, False)
            counter = float(tr._hyper_dev[5])
            for k, i in enumerate(range(first, first + replays)):
                if feed == "prefetch" and k > 0:
                    loss = tr.step_prefetched()
                else:
                    loss = tr.step(*batch(i))
                if feed == "prefetch" and k + 1 < replays:      # the next batch's copy overlaps this replay
                    tr.prefetch(*(t.pin_memory() for t in batch(i + 1, "cpu")))
                torch.cuda.synchronize()
                states[i] = dict(DP._snapshot(tr, True), loss=float(loss), replays=tr.graph_replays,
                                 iteration=tr.iteration, counter=float(tr._hyper_dev[5]),
                                 sides={n: [DP._pack(t) for t in v] for n, v in sides.items()},
                                 rec=DP._to(rec, "cpu"))
            trainable = set(tr.trainable_names)
        finally:
            conv_ops.set_mode(prev)
    del tr, sides, rec
    gc.collect()
    torch.cuda.empty_cache()
    return dict(states=states, first=first, replays=replays, after_capture=after_capture, counter=counter,
                calls=names.calls, trainable=trainable)


# ---- scoring ----------------------------------------------------------------------------------------------------
def score(monkeypatch, cid, out):
    """{replay step: dict(rows, moments, update, loss)} of a run_captured result."""
    from unflow_b200 import run
    params, B, H, W, augment, *_ = CASES[cid]
    sparams = DP.schedule(params)
    states, steps = out["states"], list(range(out["first"], out["first"] + out["replays"]))
    geff = DP.effective_gradients(states, steps)
    scores = {}
    for i in steps:
        st = states[i]
        sides = {n: [DP._unpack(t) for t in v] for n, v in st["sides"].items()}
        batch = run.synthetic_batch(B, H, W, i, 0, "cuda")
        loss, ref = float64_per_sample(monkeypatch, params, B, H, W, augment, states[i - 1]["vars"], batch, sides,
                                       st["rec"])
        scores[i] = dict(rows=DP._score(geff.pop(i), ref), moments=DP.moment_errors(states, (i,)),
                         update=DP.update_errors(states, sparams, (i,)), loss=abs(st["loss"] - loss) / abs(loss))
        del ref
        torch.cuda.empty_cache()
    return scores


def worst_geff(s):
    return max(max(s["rows"][fam]) for fam in ("weights", "biases"))


def report(title, scores, seconds):
    lines = ["%s (%.1f s)" % (title, seconds),
             "  replay  %-8s %-10s %-10s %-38s %-9s %-9s %s" % ("family", "rel L2", "max", "worst", "moments",
                                                               "update", "loss")]
    for i, s in scores.items():
        for fam in ("weights", "biases"):
            rs = s["rows"][fam]
            lines.append("  %-7d %-8s %-10.3e %-10.3e %-38s %-9.2f %-9.2f %.3e"
                         % (i, fam, max(r[1] for r in rs), max(r[2] for r in rs), max(rs)[3], s["moments"],
                            s["update"], s["loss"]))
    return "\n".join(lines)


def margins(scores):
    """{family: worst over the replays / its bound}."""
    return {"g_eff": max(worst_geff(s)[0] for s in scores.values()) / TAU_GRAD,
            "moments": max(s["moments"] for s in scores.values()) / TAU_MOMENT,
            "update": max(s["update"] for s in scores.values()) / TAU_UPDATE,
            "loss": max(s["loss"] for s in scores.values()) / TAU_LOSS}


# ---- the tests --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_captured_step_matches_float64(monkeypatch, cid):
    params, B, H, W, augment, eager, feed, calls = CASES[cid]
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    out = run_captured(monkeypatch, cid)
    t1 = time.time()
    states, first = out["states"], out["first"]
    # capture leaves the run where it found it
    assert out["after_capture"]["digest"] == states[eager]["digest"], "capture changed parameters or moments"
    assert out["counter"] == eager + 1, out["counter"]
    assert out["calls"] == calls, "entry points of the capture changed: +%s -%s" % (
        sorted(out["calls"] - calls), sorted(calls - out["calls"]))
    for k, i in enumerate(range(first, first + REPLAYS)):
        assert states[i]["replays"] == k + 1 and states[i]["iteration"] == i, (i, states[i]["replays"])
        assert states[i]["counter"] == i + 1, (i, states[i]["counter"])
    # frozen networks stay put and have no moments
    assert set(states[first]["slots"]) == out["trainable"]
    for name in set(states[0]["vars"]) - out["trainable"]:
        for i in range(first, first + REPLAYS):
            assert torch.equal(states[i]["vars"][name], states[0]["vars"][name]), name
    if augment:     # every replay draws its own augmentation: the combined masks depend on the draws alone
        masks = [states[i]["rec"].augmented[4] for i in range(first, first + REPLAYS)]
        for a in range(REPLAYS):
            for b in range(a):
                assert not torch.equal(masks[a], masks[b]), "replays %d and %d drew the same augmentation" % (b, a)
    scores = score(monkeypatch, cid, out)
    print("\n" + report("%s, %d x %dx%d, product %.1f s" % (cid, B, H, W, t1 - t0), scores, time.time() - t1))
    print("  losses %s; peak memory %.1f GB" % ([states[i]["loss"] for i in scores],
                                                 torch.cuda.max_memory_allocated() / 2 ** 30))
    for i, s in scores.items():
        for fam in ("weights", "biases"):
            assert max(s["rows"][fam])[0] <= TAU_GRAD, "replay %d %s: %s" % (i, fam, max(s["rows"][fam]))
        assert s["moments"] <= TAU_MOMENT, (i, s["moments"])
        assert s["update"] <= TAU_UPDATE, (i, s["update"])
        assert s["loss"] <= TAU_LOSS, (i, s["loss"])


@pytest.mark.gpu
@pytest.mark.parametrize("control", list(CONTROLS))
def test_bound_catches_a_captured_step_error(monkeypatch, control):
    """One error patched into the product's capture or step: the families that must catch it exceed their bounds
    by 10x."""
    _, cid, replays, families = CONTROLS[control]
    t0 = time.time()
    out = run_captured(monkeypatch, cid, control, replays)
    scores = score(monkeypatch, cid, out)
    got = margins(scores)
    print("\n" + report("%s, %s" % (cid, control), scores, time.time() - t0))
    print("%s: %s" % (control, ", ".join("%s %.0fx its bound" % (f, got[f]) for f in families)))
    for f in families:
        assert got[f] > 10, (f, got)


def test_bench_runs_these_parameters():
    """C-bench trains what bench.run_ours builds for the default --spec C."""
    from unflow_b200 import synthetic as synth
    assert C_BENCH_PARAMS == dict(synth.KITTI_PARAMS, learning_rate=1.0e-5, flownet="C")
    assert CASES["CSS-bench"][0] == dict(synth.KITTI_PARAMS, learning_rate=1.0e-5, flownet="CSS")


def test_batch_gradient_is_the_mean_of_per_sample_gradients(monkeypatch):
    """The oracle's objective in float64 on the CPU (a small FlowNetC, the KITTI loss): every variable gradient of a
    batch of 3 equals the mean over its samples to 1e-12, the L2 term included once, and so does the loss to the
    float32 rounding of the oracle's occ term.  float64_per_sample rests on this."""
    from oracle import unsupervised as ounsup
    from unflow_b200 import synthetic as synth
    import test_gpu_float64_network as N
    N._float64_ops(monkeypatch)
    monkeypatch.setattr(ounsup, "downsample", lambda t, n: R.downsample(t.contiguous(), n))
    tfv = N._variables('c', False, seed=5)
    params = dict(KITTI_PARAMS, flownet='c')
    im1, im2, _ = synth.image_pair(3, 128, 256, seed=11)

    def objective(a, b):
        leaves = {k: t.double().requires_grad_(True) for k, t in tfv.items()}
        loss = ounsup.unsupervised_loss(leaves, (a.double(), b.double()), params, normalization=N._norm())
        loss.backward()
        return float(loss.detach()), {k: v.grad for k, v in leaves.items()}

    loss, grads = objective(im1, im2)
    per = [objective(im1[b:b + 1], im2[b:b + 1]) for b in range(3)]
    mean_loss = sum(p[0] for p in per) / 3
    # the oracle sums the occ term (no gradient) over float32 masks: 3.6e-8 of this loss
    assert abs(loss - mean_loss) <= 1e-7 * abs(loss), (loss, mean_loss)
    spread = 0.0
    for k, g in grads.items():
        mean = sum(p[1][k] for p in per) / 3
        l2, mx = R.errors(g, mean)
        assert max(l2, mx) <= 1e-12, (k, l2, mx)
        spread = max(spread, max(R.errors(p[1][k], mean)[0] for p in per))
    assert spread > 1e-2, "the samples' gradients hardly differ: the test would not see a sum or a single sample"
