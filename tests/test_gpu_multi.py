"""Data parallelism on real GPUs (skipped with fewer than two): every rank ends up with the gradients of the GLOBAL
batch and replicas stay bit-identical -- with the default all-reduce between the two step graphs (eager and
graph-replayed), and with the bucketed all-reduce inside the step (CapeNetwork.set_data_parallel; opt-in:
CAPE_TEST_DP_OVERLAP=eager runs it eagerly, =1 also graph-replayed: that step completes
and returns its results, but tearing the process group down afterwards hangs, so it stays off by default)."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, use_graph, overlap, q):
    try:
        _worker_body(rank, world, port, use_graph, overlap, q)
    except BaseException as e:          # the parent must not wait for a result that will never come
        import traceback
        q.put((rank, {"error": "".join(traceback.format_exception(type(e), e, e.__traceback__))[-3000:]}))
        os._exit(1)                     # a peer may be blocked in a collective: do not wait for NCCL teardown


def _worker_body(rank, world, port, use_graph, overlap, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port), NCCL_DEBUG="WARN")
    import parity
    from cape_b200 import distributed as DP
    from cape_b200 import topology as T
    from cape_b200.network import CapeNetwork
    from cape_b200.params import NZ64_AFFINE, param_specs
    from cape_b200.synthetic import make_batch
    DP.init("nccl")
    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    cfg = dict(NZ64_AFFINE, decay_steps=10)
    specs = param_specs(cfg, [l.shape[0] for l in L], [l.shape[0] for l in L_d])
    params = parity.calibrated_params(specs, 3)
    N = 2
    order = ("x_g", "cond_g", "cond2_g", "eps", "x_d", "cond_d", "cond2_d")
    full = make_batch(N * world, cfg["nz"], seed=77)
    mine = [torch.from_numpy(full[k][rank * N:(rank + 1) * N]) for k in order]
    net = CapeNetwork(L, D, U, L_d, D_d, cfg, N, device=rank, params=params)
    allreduce = None
    if overlap:
        net.set_data_parallel(world)
    else:
        allreduce = DP.make_allreduce(world)
    net.set_inputs(*mine)
    if use_graph:
        net.train_step(step=100, update=False, allreduce=allreduce)
        torch.cuda.synchronize()
        net.capture_graphs()
    net.train_step(step=100, use_graph=use_graph, allreduce=allreduce)
    torch.cuda.synchronize()
    out = {"gg": net.PG.grad.cpu().numpy(), "gd": net.PD.grad.cpu().numpy(), "pg": net.PG.flat.cpu().numpy()}
    if rank == 0:
        # the same global batch on one GPU, no data parallelism
        ref = CapeNetwork(L, D, U, L_d, D_d, cfg, N * world, device=0, params=params)
        ref.set_inputs(*[torch.from_numpy(full[k]) for k in order])
        ref.train_step(step=100)
        torch.cuda.synchronize()
        out.update(ref_gg=ref.PG.grad.cpu().numpy(), ref_gd=ref.PD.grad.cpu().numpy(), ref_pg=ref.PG.flat.cpu().numpy())
    q.put((rank, out))
    import torch.distributed as dist
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("use_graph,overlap", [(False, False), (True, False), (False, True), (True, True)])
def test_data_parallel_step_equals_global_batch(use_graph, overlap):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    want = os.environ.get("CAPE_TEST_DP_OVERLAP", "0")       # "1": eager and graph-replayed, "eager": eager only
    if overlap and not (want == "1" or (want == "eager" and not use_graph)):
        pytest.skip("bucketed in-step all-reduce: opt-in (CAPE_TEST_DP_OVERLAP=1|eager)")
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, use_graph, overlap, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(world):
            rank, out = q.get(timeout=240)
            res[rank] = out
            assert "error" not in out, "rank %d failed:\n%s" % (rank, out["error"])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:                 # never leave a rank behind (it would hold its GPU until the box is recycled)
            if p.is_alive():
                p.kill()
    rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
    r0, r1 = res[0], res[1]
    assert np.array_equal(r0["gg"], r1["gg"]) and np.array_equal(r0["pg"], r1["pg"])     # replicas stay identical
    # The single-GPU reference tiles the global batch differently (row tiles straddle other samples, the weight gradients
    # split their row range differently), so tensor-core accumulation order differs at the 1e-5 level and the VAE's
    # exp(logvar) amplifies it: a missing or misplaced all-reduce shows up as an O(1) error, not as 1e-4.
    e_gg, e_gd, e_pg = rel(r0["gg"], r0["ref_gg"]), rel(r0["gd"], r0["ref_gd"]), rel(r0["pg"], r0["ref_pg"])
    print("data-parallel vs global batch: generator grads %.2e, discriminator grads %.2e, parameters %.2e" % (e_gg, e_gd, e_pg))
    assert e_gg < 3e-4 and e_gd < 3e-4
    assert e_pg < 1e-6
