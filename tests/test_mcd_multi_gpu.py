"""Data-parallel TrainStep with ens_DA='MCD' on 2 GPUs (the library's peer all-reduce): the mean of the shard gradients
equals the single-GPU gradient of the global batch, classifier 2 and pass 2's contribution included.  Needs >= 2 CUDA
devices; skipped otherwise."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ta3n_oracle as orc

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")]

B_LOCAL = 24
MU = 0.7


def _cfg():
    return orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0, ens_DA="MCD")


def _build(dev):
    from ta3n_b200.models import VideoModel
    cfg = _cfg()
    m = VideoModel(cfg.num_class, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=512,
                   dropout_i=0.0, dropout_v=0.0, ens_DA="MCD", partial_bn=False, verbose=False)
    params = orc.init_params(cfg, seed=99)
    g = torch.Generator().manual_seed(100)
    for k in params:
        if params[k].dtype.is_floating_point and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    m.load_state_dict(params)
    return m.to(dev).train()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        import ta3n_b200
        from ta3n_b200.parallel import shard_rows
        from ta3n_b200.train import TrainStep
        ta3n_b200.set_gemm_engine("fp32")
        xs, xt, labels = orc.synthetic_batch(world * B_LOCAL, _cfg())
        sl = shard_rows(world * B_LOCAL, rank, world)
        step = TrainStep(_build(dev), B_LOCAL, B_LOCAL, (0.75, 0.75, 0.5), gamma=0.0, use_graph=True,
                         allreduce="peer", mu=MU)
        assert step.ar is not None
        step(xs[sl], xt[sl], labels[sl])
        torch.cuda.synchronize()
        if rank == 0:
            q.put(step.flat_grad.cpu().numpy())
    finally:
        dist.destroy_process_group()


def test_mcd_peer_allreduce_matches_global_batch():
    import ta3n_b200
    from ta3n_b200.train import TrainStep
    ta3n_b200.set_gemm_engine("fp32")
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = torch.from_numpy(q.get(timeout=300))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    xs, xt, labels = orc.synthetic_batch(world * B_LOCAL, _cfg())
    # gamma = 0: every loss term is a plain mean over rows, so the mean of the shard means is the global mean
    ref = TrainStep(_build(torch.device("cuda", 0)), world * B_LOCAL, world * B_LOCAL, (0.75, 0.75, 0.5), gamma=0.0,
                    use_graph=True, mu=MU)
    ref(xs, xt, labels)
    torch.cuda.synchronize()
    want = ref.flat_grad.cpu()
    err = ((got.double() - want.double()).norm() / want.double().norm()).item()
    assert err < 1e-4, err
    assert float(ref.grad_views[-2].norm()) > 0         # classifier 2's slot is part of the compared bucket
