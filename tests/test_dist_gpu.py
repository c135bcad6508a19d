"""2-GPU NCCL test of the track-sharded LM (skipped on boxes with one GPU): both ranks must reproduce the
single-GPU trajectory, hold identical cameras and own their slice of the points."""
import os
import socket

import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.helpers import ba_case

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q, use_fabric=False):
    import torch
    import torch.distributed as dist
    from vggsfm_b200 import bundle_adjustment as ba
    from vggsfm_b200.dist import AllReduceHook, shard_range
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    c = ba_case(12, 512, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=3)
    lo, hi = shard_range(512, rank, world)
    t = lambda a, dt=None: (torch.from_numpy(np.ascontiguousarray(a)).to(dt) if dt else torch.from_numpy(np.ascontiguousarray(a))).to(dev).contiguous()
    poses, intr, pts = t(c["poses"]), t(c["intr"]), t(c["points"][lo:hi])
    opt = ba.default_options()
    opt.max_num_iterations = 8
    fabric = None
    if use_fabric:
        from vggsfm_b200.dist import FabricBuffer
        fabric = FabricBuffer(12, c["model"], c["mode"], dev)
    hook = AllReduceHook(fabric=fabric)
    s = ba.lm_solve(t(c["uv"][:, lo:hi], torch.float32), t(c["mask"][:, lo:hi].astype(np.uint8)), poses, intr, pts,
                    c["model"], c["mode"], options=opt, allreduce=hook, want_trace=True)
    q.put((rank, poses.cpu().numpy(), intr.cpu().numpy(), pts.cpu().numpy(), s.iterations, s.final_cost,
           s.trace.numpy().copy(), hook.calls, hook.barriers, bool(fabric is not None and fabric.ok)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("use_fabric", [False, True], ids=["nccl_allreduce", "fabric_v2_reduce_scatter"])
def test_two_gpu_sharded_lm_matches_single_gpu(use_fabric):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from vggsfm_b200 import bundle_adjustment as ba
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, use_fabric)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    c = ba_case(12, 512, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=3)
    dev = torch.device("cuda:0")
    t = lambda a, dt=None: (torch.from_numpy(np.ascontiguousarray(a)).to(dt) if dt else torch.from_numpy(np.ascontiguousarray(a))).to(dev).contiguous()
    poses, intr, pts = t(c["poses"]), t(c["intr"]), t(c["points"])
    opt = ba.default_options()
    opt.max_num_iterations = 8
    s = ba.lm_solve(t(c["uv"], torch.float32), t(c["mask"].astype(np.uint8)), poses, intr, pts, c["model"], c["mode"],
                    options=opt, want_trace=True)
    for rank, p, i, x, its, cost, tr, calls, barriers, fabric_ok in res:
        lo, hi = (0, 256) if rank == 0 else (256, 512)
        assert its == s.iterations
        if fabric_ok:
            assert calls == 0 and barriers == 0      # no NCCL call, no host callback: everything is csrc/fabric.cu kernels
        else:
            assert calls >= 2 * its
        if use_fabric and not fabric_ok:
            pytest.skip("no NVSwitch multicast on this box")
        assert abs(cost - s.final_cost) <= 1e-9 * s.final_cost
        assert np.allclose(tr[:, 2], s.trace.numpy()[:, 2], rtol=1e-8)
        assert np.abs(p - poses.cpu().numpy()).max() < 1e-8
        assert np.abs(x - pts.cpu().numpy()[lo:hi]).max() < 1e-8
    assert np.array_equal(res[0][1], res[1][1])      # identical cameras on both ranks (same reduced system, same solve)
