"""Data-parallel training step: forward + loss + backward + gradient all-reduce + Adam.

Counterpart of the reference Trainer's hot loop (src/e2eflow/core/train.py:147-185 graph
construction, :222-251 ``sess.run([train_op, loss_])``, :388-422 ``average_gradients``) -- only
the step itself; the reference's session / checkpoint / summary / eval scaffolding is TF specific
and outside the hot path (SURVEY.md section 8f, row N1).

Design (one process per GPU):
  * every trainable variable is a view into ONE flat fp32 buffer, every gradient a view into a
    second one -> the tower-gradient mean of the reference (concat + reduce_mean on the CPU,
    train.py:388-422) is a single ``all_reduce`` over NCCL / NVLink on the flat gradient buffer,
    and the optimiser is a single fused Adam kernel (csrc/adam.cu) that also clears the gradients;
  * unlike the reference (whose towers all consume the same dequeued batch, train.py:169,191)
    each rank gets its own shard of the global batch; the averaged gradient equals the 1-GPU
    gradient of the concatenated batch;
  * learning-rate schedule: ``learning_rate`` halved every ``decay_interval`` iterations after
    ``decay_after`` (train.py:225-244).
"""
import torch
import torch.distributed as dist

from ... import _native
from ..._native import check
from .flownet import FlowNetVariables
from .supervised import supervised_loss
from .unsupervised import unsupervised_loss


def learning_rate_at(decay_iters, params):
    """Host-side LR schedule of the reference training loop (train.py:225-244).

    ``decay_iters`` = number of iterations already done (the reference's
    ``local_i + iter_offset``, 0 for the first step)."""
    if 'manual_decay_lrs' in params and 'manual_decay_iters' in params:
        decay_index = 0
        iter_counter = 0
        for decay_i, manual_decay_iter in enumerate(params['manual_decay_iters']):
            iter_counter += manual_decay_iter
            if decay_iters <= iter_counter:
                decay_index = decay_i
                break
        return params['manual_decay_lrs'][decay_index]
    lr = params.get('learning_rate', 1.0e-4)
    decay_interval = params.get('decay_interval')
    if not decay_interval:
        return lr
    decay_after = params.get('decay_after', 0)
    if decay_iters >= decay_after:
        decay_minimum = decay_after / decay_interval
        decay = (decay_iters // decay_interval) - decay_minimum
        return lr / (2 ** decay)
    return lr


def l2_mask_bytes(n, offsets, numels, regularised):
    """Mask of the regularised elements of the flat parameter buffer in the form csrc/adam.cu reads:
    (per-element uint8 flags, one byte per float4 with bit k = element 4 * i + k).  ``n`` is a multiple of 4."""
    isw = torch.zeros(n, dtype=torch.uint8)
    for off, k, reg in zip(offsets, numels, regularised):
        if reg:
            isw[off:off + k] = 1
    q = isw.view(-1, 4)
    return isw, (q[:, 0] | (q[:, 1] << 1) | (q[:, 2] << 2) | (q[:, 3] << 3)).contiguous()


def _batch_and_option(args, option):
    """Split positional arguments into the batch tensors and a trailing non-tensor option (the
    ``lr`` of ``step(im1, im2, lr)``, the ``warmup`` of ``capture(im1, im2, warmup)``)."""
    if args and not torch.is_tensor(args[-1]):
        if option is not None:
            raise TypeError("the option was given twice")
        return tuple(args[:-1]), args[-1]
    return tuple(args), option


class Trainer:
    def __init__(self, params, normalization, device, variables=None, seed=1234,
                 loss_fn=unsupervised_loss, process_group=None, augment=False, supervised=False):
        """``supervised``: train on ``supervised_loss`` (fine-tuning on ground truth, the reference's
        ``Trainer(..., supervised=True)``, train.py:98-112); the batch is then
        ``(im1, im2, flow_gt, mask_gt)`` instead of ``(im1, im2)``.  ``step``, ``capture``, ``prefetch``
        and ``step_prefetched`` take the batch tensors as positional arguments, however many there are.

        ``augment``: run the reference's training-time augmentation (random_affine x3 +
        random_photometric, unsupervised.py:39-60) inside every step, as the reference Trainer does
        (``loss_fn(batch, params, normalization)`` with the default ``augment=True``,
        train.py:160,169).  run.py trains with it on; bench.py and the parity tests keep it off
        (random draws cannot be parity-pinned).  The draws come from the device generator so the
        step stays capturable in a CUDA graph."""
        self.augment = bool(augment)
        if self.augment:
            from . import augment as _aug
            _aug.set_device_rng(True)
        self.params = dict(params)
        self.normalization = normalization
        self.device = torch.device(device)
        self.supervised = bool(supervised)
        self.loss_fn = supervised_loss if self.supervised else loss_fn
        self.pg = process_group
        self.world_size = dist.get_world_size(process_group) if dist.is_initialized() else 1
        spec = self.params.get('flownet', 'S')
        if variables is None:
            variables = FlowNetVariables(spec, self.params.get('full_res'), seed=seed)
        self.variables = variables.to(self.device)
        # Only the final network of a stack is trained unless train_all (config.ini:55-58).
        n_nets = len(spec)
        if self.params.get('train_all') or n_nets == 1:
            scopes = list(self.variables.kinds)
        else:
            scopes = self.variables.scopes_of_net(n_nets - 1)
        trainable, names = [], []
        for sc in scopes:
            w, b = self.variables.weights(sc)
            trainable += [w, b]
            names += [sc + '/weights', sc + '/biases']
        self.trainable_names = names
        train_ids = {id(p) for p in trainable}
        for p in self.variables.parameters():
            p.requires_grad_(id(p) in train_ids)
        self.trainable = trainable
        self._flatten()
        self.iteration = 0
        self._graph = None
        # keep the tracked images of every step for image summaries (unsupervised.tracked_images)
        self.track_images = False
        # L2 regularisation gradient inside the Adam kernel (CUDA only; on the CPU autograd forms it).
        # flat_grad then holds the gradient of the data terms only -- l2_gradient() is the missing part.
        self.l2_mask = None
        self.l2_scale = float(self.variables.L2_SCALE)
        if self.device.type == 'cuda':
            isw, packed = l2_mask_bytes(self.flat_param.numel(), self._offsets, [p.numel() for p in self.trainable],
                                        [name.endswith('/weights') for name in self.trainable_names])
            self.l2_mask = packed.to(self.device)
            self._l2_elements = isw.to(self.device)
            self.variables.l2_in_optimizer = True

    def _flatten(self):
        n = sum(p.numel() for p in self.trainable)
        npad = (n + 3) // 4 * 4
        self.flat_param = torch.zeros(npad, device=self.device, dtype=torch.float32)
        self.flat_grad = torch.zeros(npad, device=self.device, dtype=torch.float32)
        self.adam_m = torch.zeros(npad, device=self.device, dtype=torch.float32)
        self.adam_v = torch.zeros(npad, device=self.device, dtype=torch.float32)
        off = 0
        self._offsets = []
        with torch.no_grad():
            for p in self.trainable:
                k = p.numel()
                pv = self._view_like(self.flat_param[off:off + k], p)
                pv.copy_(p)
                p.data = pv
                p.grad = self._view_like(self.flat_grad[off:off + k], p)
                self._offsets.append(off)
                off += k
        self.num_params = n

    @staticmethod
    def _view_like(flat_seg, p):
        """A view of the flat segment with p's shape; 4-D weights keep their NHWC memory order."""
        if p.dim() == 4:
            a, b, kh, kw = p.shape
            return flat_seg.view(a, kh, kw, b).permute(0, 3, 1, 2)
        return flat_seg.view_as(p)

    # -- optimizer state in the reference's checkpoint naming --------------------------------------
    def adam_slots(self):
        """{variable name: (m, v)} in TF layout -- the ``<name>/Adam`` and ``<name>/Adam_1`` slot
        variables tf.train.AdamOptimizer creates next to each trained variable (train.py:151-152)."""
        out = {}
        for name, p, off in zip(self.trainable_names, self.trainable, self._offsets):
            pair = []
            for flat in (self.adam_m, self.adam_v):
                t = self._view_like(flat[off:off + p.numel()], p)
                if p.dim() == 4:
                    t = t.permute(2, 3, 1, 0)
                pair.append(t.detach().clone(memory_format=torch.contiguous_format).cpu().numpy())
            out[name] = tuple(pair)
        return out

    def load_adam_slots(self, slots):
        """Inverse of ``adam_slots``; variables without an entry keep zero moments."""
        with torch.no_grad():
            for name, p, off in zip(self.trainable_names, self.trainable, self._offsets):
                if name not in slots:
                    continue
                for flat, value in zip((self.adam_m, self.adam_v), slots[name]):
                    t = torch.as_tensor(value, dtype=torch.float32)
                    if p.dim() == 4:
                        t = t.permute(3, 2, 0, 1)
                    self._view_like(flat[off:off + p.numel()], p).copy_(t)

    def broadcast_variables(self, src=0):
        if self.world_size > 1:
            dist.broadcast(self.flat_param, src, group=self.pg)

    def loss(self, *batch):
        from . import unsupervised
        unsupervised.track_images = self.track_images
        return self.loss_fn(tuple(batch), self.params, self.normalization, augment=self.augment,
                            variables=self.variables)

    def reduce_gradients(self):
        """Mean of the gradients over ranks: ONE all-reduce on the flat buffer (NCCL over NVLink on
        GPUs).  Returns the factor still to be applied (folded into the Adam kernel)."""
        if self.world_size > 1:
            dist.all_reduce(self.flat_grad, op=dist.ReduceOp.SUM, group=self.pg)
            return 1.0 / self.world_size
        return 1.0

    def l2_gradient(self):
        """The regularisation gradient the Adam kernel adds (zeros when autograd forms it instead)."""
        if self.l2_mask is None:
            return torch.zeros_like(self.flat_param)
        return self.l2_scale * self.flat_param * self._l2_elements

    def apply_update(self, lr, grad_scale=1.0):
        if self.flat_param.device.type != "cuda":
            raise RuntimeError("the Adam update is a CUDA kernel (csrc/adam.cu); no CPU fallback")
        from ..ops import kernel_timer
        with torch.cuda.device(self.device), kernel_timer.span("adam", 32 * self.flat_param.numel()):
            check(_native.lib().unflow_adam_step_l2(
                self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.adam_m.data_ptr(),
                self.adam_v.data_ptr(), self.flat_param.numel(), float(lr), 0.9, 0.999, 1e-8,
                self.iteration, float(grad_scale), 1,
                self.l2_mask.data_ptr() if self.l2_mask is not None else None, self.l2_scale,
                torch.cuda.current_stream().cuda_stream), "adam_step")

    def _set_hyper(self, lr, step):
        """(rare, synchronous) host -> device update of [lr, beta1, beta2, eps, grad_scale, step]."""
        vals = torch.tensor([lr, 0.9, 0.999, 1e-8, 1.0 / self.world_size, float(step), 0.0, 0.0])
        self._hyper_dev.copy_(vals.to(self.device))
        torch.cuda.synchronize(self.device)
        self._hyper_lr = lr

    def _step_impl(self, *batch):
        """forward + loss + backward + gradient mean + Adam, hyper-parameters from device memory."""
        loss = self.loss(*batch)
        loss.backward()
        self.reduce_gradients()
        from ..ops import kernel_timer
        with torch.cuda.device(self.device), kernel_timer.span("adam", 32 * self.flat_param.numel()):
            check(_native.lib().unflow_adam_step_dev_l2(
                self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.adam_m.data_ptr(),
                self.adam_v.data_ptr(), self.flat_param.numel(), self._hyper_dev.data_ptr(), 1,
                self.l2_mask.data_ptr() if self.l2_mask is not None else None, self.l2_scale,
                torch.cuda.current_stream().cuda_stream), "adam_step")
        return loss.detach()

    def capture(self, *batch, warmup=None):
        """Capture the whole training step (several hundred kernels: cuDNN convs, the hand-written
        kernels, the NCCL all-reduce, Adam) into ONE CUDA graph.  Later ``step`` calls copy the batch
        into the static input buffers, refresh the hyper-parameter vector and replay the graph, so
        the host launches one graph instead of ~800 kernels per step."""
        batch, warmup = _batch_and_option(batch, warmup)
        warmup = 3 if warmup is None else warmup
        assert self.flat_param.is_cuda
        self._hyper_dev = torch.zeros(8, device=self.device, dtype=torch.float32)
        self._static = [t.to(self.device).clone() for t in batch]     # the graph's input buffers
        self._static_im1, self._static_im2 = self._static[0], self._static[1]
        moments = (self.adam_m.clone(), self.adam_v.clone())   # restored below (resumed runs carry state)
        self._set_hyper(0.0, 1.0)                         # lr = 0 while warming up / capturing
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):                       # eager warm-up (cuDNN autotune, caches)
                self._step_impl(*self._static)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(self.device)
        n0 = _native.launch_count()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._static_loss = self._step_impl(*self._static)
        self._graph_launches = _native.launch_count() - n0
        # the tracked values of the captured step live in the graph's memory: every replay rewrites them
        from . import unsupervised
        self._graph_tracked = (dict(unsupervised.tracked), dict(unsupervised.tracked_params),
                               dict(unsupervised.tracked_images))
        torch.cuda.synchronize(self.device)
        # lr = 0 left the parameters alone but fed the moments: put them back, reset the step counter
        self.adam_m.copy_(moments[0]); self.adam_v.copy_(moments[1]); self.flat_grad.zero_()
        self._set_hyper(learning_rate_at(self.iteration, self.params), self.iteration + 1)
        self._graph = graph
        self.graph_replays = 0
        return self

    # -- input prefetch (opt-in; graph mode) -----------------------------------------------------
    def prefetch(self, *host_batch):
        """Start copying the NEXT batch (pinned host tensors) into staging buffers on a copy stream;
        it overlaps the step that is currently running.  Pair with ``step_prefetched``."""
        assert self._graph is not None, "prefetch() needs a captured step (capture())"
        if len(host_batch) != len(self._static):
            raise ValueError("prefetch: %d tensors for a step captured with %d"
                             % (len(host_batch), len(self._static)))
        if getattr(self, '_copy_stream', None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._stage = [torch.empty_like(t) for t in self._static]
            self._stage_im1, self._stage_im2 = self._stage[0], self._stage[1]
            self._stage_free = None
        cs = self._copy_stream
        if self._stage_free is not None:
            cs.wait_event(self._stage_free)            # the previous contents have been consumed
        with torch.cuda.stream(cs):
            for dst, src in zip(self._stage, host_batch):
                dst.copy_(src, non_blocking=True)
            self._stage_ready = torch.cuda.Event()
            self._stage_ready.record(cs)

    def step_prefetched(self, lr=None):
        """``step`` on the batch handed to the last ``prefetch`` call: the compute stream waits for the
        staged copy, moves it into the graph's static input buffers (device to device) and replays."""
        self.iteration += 1
        if lr is None:
            lr = learning_rate_at(self.iteration - 1, self.params)
        if lr != self._hyper_lr:
            self._set_hyper(lr, self.iteration)
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(self._stage_ready)
        for dst, src in zip(self._static, self._stage):
            dst.copy_(src, non_blocking=True)
        self._stage_free = torch.cuda.Event()
        self._stage_free.record(cur)
        self._graph.replay()
        self.graph_replays += 1
        return self._static_loss

    def step(self, *batch, lr=None):
        """One optimisation step on this rank's shard (``step(im1, im2)``, or
        ``step(im1, im2, flow_gt, mask_gt)`` when supervised); returns the (local) loss tensor."""
        batch, lr = _batch_and_option(batch, lr)
        self.iteration += 1
        if lr is None:
            lr = learning_rate_at(self.iteration - 1, self.params)
        if self._graph is not None:
            if lr != self._hyper_lr:                      # the schedule moved: rewrite lr (rare)
                self._set_hyper(lr, self.iteration)
            if len(batch) != len(self._static):
                raise ValueError("step: %d tensors for a step captured with %d" % (len(batch), len(self._static)))
            for dst, src in zip(self._static, batch):
                dst.copy_(src, non_blocking=True)
            self._graph.replay()
            self.graph_replays += 1
            return self._static_loss
        loss = self.loss(*batch)
        loss.backward()   # accumulates into the flat gradient views
        scale = self.reduce_gradients()
        self.apply_update(lr, scale)
        return loss.detach()

    def tracked(self):
        """The last step's tracked values as (losses, params, images): {op name: tensor or float} in
        the order the reference creates the ops, {op name: float} and {op name: (tensor, to_image)}.
        After ``capture`` these are the captured step's outputs, which every replay refreshes."""
        if self._graph is not None:
            return self._graph_tracked
        from . import unsupervised
        return unsupervised.tracked, unsupervised.tracked_params, unsupervised.tracked_images

    def summary_scalars(self):
        """{op name: float} of the last step's tracked losses, read with one device-to-host copy."""
        return read_scalars(self.tracked()[0])


def read_scalars(values):
    """{name: float} of a dict of scalar tensors and Python numbers; the tensors are stacked on their
    device and copied to the host at once."""
    names = [k for k, v in values.items() if torch.is_tensor(v)]
    out = {k: float(v) for k, v in values.items() if not torch.is_tensor(v)}
    if names:
        host = torch.stack([values[k].reshape(()).float() for k in names]).cpu()
        out.update(zip(names, host.tolist()))
    return {k: out[k] for k in values}


def evaluate(variables, params, normalization, examples, eval_size=(384, 1280), loss_averages=None, pages=None):
    """The checkpoint-evaluation loop of the reference Trainer (train.py:265-385) without the TF
    session / summary scaffolding.

    ``examples``: iterable of ``(im1, im2, flow_occ, mask_occ, flow_noc, mask_noc)`` with float
    tensors ``[1,h,w,C]`` on the device (the layout ``einput.input_train_2012()`` yields).
    Each pair is resized to ``eval_size`` (384x1280, train.py:274-275) with the TF1 bilinear kernel,
    run through ``unsupervised_loss(augment=False, return_flow=True)``, the flow is resized back and
    rescaled (``resize_output_flow``), and AEE / outlier-% are averaged over the examples for the
    'occluded' (all valid) and 'non-occluded' masks (train.py:314-321).  Returns the dict of
    averages plus the last example's visualisation tensors (train.py:290-293).  ``loss_averages``: a
    dict that receives every tracked loss of ``unsupervised_loss`` averaged over the examples
    (train.py:323-328), {op name: float}.  ``pages``: a ``pages.Tiles`` that receives every example's
    visualisation tensors as uint8 (the reference's interactive plot, train.py:378-384)."""
    from . import flow_util, tf_image
    from .flow_io import resize_output_flow
    from .image_warp import image_warp
    from .losses import DISOCC_THRESH, create_outgoing_mask, occlusion
    from ..ops import forward_warp
    sums, loss_sums, n, images = {}, {}, 0, None
    rh, rw = eval_size
    with torch.no_grad():
        for (im1, im2, flow_occ, mask_occ, flow_noc, mask_noc) in examples:
            h, w = im1.shape[1], im1.shape[2]
            a = tf_image.resize_bilinear(im1, [rh, rw])
            b = tf_image.resize_bilinear(im2, [rh, rw])
            _, flow, flow_bw = unsupervised_loss((a, b), params, normalization, augment=False,
                                                 return_flow=True, variables=variables)
            if loss_averages is not None:
                from .unsupervised import tracked
                for k, v in read_scalars(tracked).items():
                    loss_sums[k] = loss_sums.get(k, 0.0) + v
            flow = resize_output_flow(flow, h, w).contiguous()
            flow_bw = resize_output_flow(flow_bw, h, w).contiguous()
            for name, gt, mask in (('occluded', flow_occ, mask_occ), ('non-occluded', flow_noc, mask_noc)):
                sums['AEE/' + name] = sums.get('AEE/' + name, 0.0) + float(flow_util.flow_error_avg(gt, flow, mask))
                sums['outliers/' + name] = sums.get('outliers/' + name, 0.0) + float(
                    flow_util.outlier_pct(gt, flow, mask))
            n += 1
            images = {'warped image': image_warp(im1.contiguous(), flow) / 255,
                      'flow': flow_util.flow_to_color(flow),
                      'occ': 1 - (1 - occlusion(flow, flow_bw)[0]) * create_outgoing_mask(flow),
                      'reverse disocc': forward_warp(flow_bw) < DISOCC_THRESH,
                      'flow error': flow_util.flow_error_image(flow, flow_occ, mask_occ, mask_noc)}
            if pages is not None and pages.wants_more():
                from .pages import to_uint8
                pages.add(list(images), [to_uint8(v * 255) for v in images.values()])
    out = {k: v / max(n, 1) for k, v in sums.items()}
    out['num_examples'] = n
    if loss_averages is not None:
        loss_averages.update({k: v / max(n, 1) for k, v in loss_sums.items()})
    return out, images
