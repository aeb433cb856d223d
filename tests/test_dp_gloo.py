"""World-size-2 test of the data-parallel host logic on CPU (gloo): flat parameter / gradient
buffers, one all-reduce, and "N ranks == 1 rank on the concatenated batch" (SURVEY.md R4/8e)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _toy_loss(batch, params, normalization, augment, variables):
    """FlowNetS forward (no custom op -> runs on CPU) + a smooth loss; mean over the shard."""
    from unflow_b200.e2eflow.core.flownet import flownet
    im1, im2 = batch
    flows = flownet(im1, im2, 's', variables=variables)[0]
    return sum((f ** 2).mean() for f in flows) + variables.regularization_loss()


def _data(n):
    g = torch.Generator().manual_seed(7)
    return torch.rand(n, 64, 64, 3, generator=g) - 0.5, torch.rand(n, 64, 64, 3, generator=g) - 0.5


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    from unflow_b200.e2eflow.core.train import Trainer
    tr = Trainer(dict(flownet='s'), None, "cpu", seed=rank * 17 + 3, loss_fn=_toy_loss)
    tr.broadcast_variables(0)                       # ranks start from rank 0's weights
    im1, im2 = _data(4)
    sl = slice(2 * rank, 2 * rank + 2)              # distinct shard per rank
    loss = tr.loss(im1[sl], im2[sl])
    loss.backward()
    scale = tr.reduce_gradients()
    single = tr.flat_grad * scale
    if rank == 0:
        torch.save({"grad": single, "param": tr.flat_param.clone(), "n": tr.num_params}, out)
    with pytest.raises(RuntimeError):
        tr.apply_update(1e-4, scale)                # the optimiser kernel is CUDA only: loud failure
    dist.destroy_process_group()


def test_two_rank_all_reduce_equals_single_rank_on_concatenated_batch(tmp_path):
    out = str(tmp_path / "dp.pt")
    mp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    got = torch.load(out)
    from unflow_b200.e2eflow.core.train import Trainer
    tr = Trainer(dict(flownet='s'), None, "cpu", seed=3, loss_fn=_toy_loss)
    assert torch.equal(tr.flat_param, got["param"])       # broadcast delivered rank 0's weights
    assert tr.num_params == got["n"]
    im1, im2 = _data(4)
    # mean over 4 == mean of the two shard means (equal shard sizes); the regulariser is identical
    loss = 0.5 * (tr.loss(im1[:2], im2[:2]) + tr.loss(im1[2:], im2[2:]))
    loss.backward()
    err = float((tr.flat_grad - got["grad"]).norm() / tr.flat_grad.norm())
    assert err < 1e-5, err


def test_flat_views_alias_parameters():
    from unflow_b200.e2eflow.core.train import Trainer, learning_rate_at
    tr = Trainer(dict(flownet='ss'), None, "cpu", seed=0, loss_fn=_toy_loss)
    # only the last network of the stack is trainable (config.ini:55-58)
    names = {n for n, p in tr.variables.named_parameters() if p.requires_grad}
    assert names and all("stack_1_flownet" in n for n in names)
    w, _ = tr.variables.weights("stack_1_flownet/flownet_s/conv1")
    tr.flat_param.zero_()
    assert float(w.abs().sum()) == 0.0
    tr.flat_grad.fill_(2.0)
    assert float(w.grad.mean()) == 2.0
    p = dict(learning_rate=1e-4, decay_after=10, decay_interval=5)   # train.py:237-244
    assert learning_rate_at(9, p) == 1e-4 and learning_rate_at(10, p) == 1e-4
    assert learning_rate_at(15, p) == 5e-5 and learning_rate_at(21, p) == 2.5e-5
    m = dict(manual_decay_iters=[3, 2], manual_decay_lrs=[1e-5, 5e-6])  # train.py:228-236
    assert [learning_rate_at(i, m) for i in range(6)] == [1e-5, 1e-5, 1e-5, 1e-5, 5e-6, 5e-6]
