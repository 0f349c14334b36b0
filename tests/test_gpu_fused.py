"""GPU tests of the fused path (pytest -m gpu on an H100).

Numerics oracle: plain PyTorch fp32 SGD on the concatenated batch.  Multi-rank cases run one
process per rank; with a single GPU all ranks share cuda:0 (CUDA IPC works between processes on one
device), with >= 2 GPUs each rank gets its own device and the data moves over NVLink.
"""

import pytest
import torch
import torch.nn as nn

from _mp import run_ranks
from test_dear_equivalence import CASES, data, make_model, reference_run

pytestmark = pytest.mark.gpu


def gpu_worker(rank, world, case, steps, per_rank, threshold, dtype_name):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    assert ops.native_path() is not None
    dev = dear.device()
    model = make_model().to(dev)
    model.eval()
    if dtype_name == "bf16":
        model = model.to(torch.bfloat16)
    opt = torch.optim.SGD(model.parameters(), lr=0.05, **case)
    opt = dear.DistributedOptimizer(opt, model, threshold=threshold, verbose=False)
    dear.broadcast_parameters(model.state_dict(), 0)
    for t in range(steps):
        x, y = data(t, world * per_rank)
        x, y = x[rank * per_rank:(rank + 1) * per_rank].to(dev), y[rank * per_rank:(rank + 1) * per_rank].to(dev)
        if dtype_name == "bf16":
            x = x.to(torch.bfloat16)
        opt.zero_grad()
        nn.functional.cross_entropy(model(x).float(), y).backward()
        opt.step()
    opt.synchronize()
    dear.communicator().check_status()
    return [p.detach().float().cpu() for p in model.parameters()], dear.communicator().launches()


def _env():
    # several ranks may have to share one GPU on the test box
    return {"DEAR_SPIN_TIMEOUT_S": "15"}


@pytest.mark.parametrize("case", [CASES[0], CASES[2], CASES[3]])
def test_single_gpu_fused_sgd_matches_torch(case):
    ref = reference_run(case, 4, 1, 8)
    outs = run_ranks(gpu_worker, world=1, backend="b200", args=(case, 4, 8, 0.001, "fp32"), extra_env=_env())
    params, launches = outs[0]
    assert launches > 0
    for a, b in zip(params, ref):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_rank_fused_matches_torch(world):
    ngpu = torch.cuda.device_count()
    if (ngpu > 1 and ngpu < world) or (world == 8 and ngpu < 8):
        pytest.skip("needs %d GPUs (2 and 4 ranks may also share exactly one GPU)" % world)
    case = CASES[2]
    ref = reference_run(case, 3, world, 2)
    outs = run_ranks(gpu_worker, world=world, backend="b200", args=(case, 3, 2, 0.001, "fp32"), extra_env=_env(),
                     timeout=300)
    for params, launches in outs:
        assert launches > 0
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    for a, b in zip(outs[0][0], outs[-1][0]):
        assert torch.equal(a, b)


def test_bf16_params_fp32_master():
    case = dict(momentum=0.9)
    ref = reference_run(case, 3, 2, 4)
    outs = run_ranks(gpu_worker, world=2 if torch.cuda.device_count() != 1 or True else 1, backend="b200",
                     args=(case, 3, 4, 0.001, "bf16"), extra_env=_env(), timeout=300)
    for params, _ in outs:
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, rtol=5e-2, atol=5e-2)
    for a, b in zip(outs[0][0], outs[-1][0]):
        assert torch.equal(a, b)


def comm_worker(rank, world):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    comm = dear.communicator()
    res = {}
    t = torch.arange(1000, device=dev, dtype=torch.float32) * (rank + 1)
    dear.allreduce(t)
    res["allreduce"] = t.cpu()
    b = torch.arange(7, device=dev, dtype=torch.int64) * (rank + 5)
    dear.broadcast_(b, world - 1)
    res["bcast"] = b.cpu()
    big = torch.full((3_000_001,), float(rank + 1), device=dev)
    h = comm.allReduceRSAG(big[:3_000_000 // world * world], 1.0)
    comm.syncStream(h)
    res["rsag"] = big[:4].cpu()
    g = dear.allgather(torch.full((5,), float(rank), device=dev))
    res["allgather"] = g.cpu()
    h = comm.allReduceRB(t, 1.0)
    comm.syncStream(h)
    res["rb"] = t[:3].cpu()
    send = torch.full((9,), float(rank), device=dev)
    recv = torch.empty_like(send)
    h = comm.sendrecv(send, recv, (rank + 1) % world)
    comm.syncStream(h)
    res["sendrecv"] = recv.cpu()
    comm.check_status()
    return res


def test_general_collectives():
    world = 2
    outs = run_ranks(comm_worker, world=world, backend="b200", extra_env=_env(), timeout=300)
    s = sum(range(1, world + 1))
    for r, res in enumerate(outs):
        torch.testing.assert_close(res["allreduce"], torch.arange(1000.) * s / world)
        assert torch.equal(res["bcast"], torch.arange(7) * (world - 1 + 5))
        torch.testing.assert_close(res["rsag"], torch.full((4,), float(s)))
        torch.testing.assert_close(res["allgather"], torch.arange(world).repeat_interleave(5).float())
        torch.testing.assert_close(res["rb"], (torch.arange(1000.) * s / world)[:3] * world)
        torch.testing.assert_close(res["sendrecv"], torch.full((9,), float((r + 1) % world)))


def graph_worker(rank, world, use_graph, overlap=False, adam=False):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200.utils.train import TrainStep
    dev = dear.device()
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 10)).to(dev)
    if adam:
        opt = torch.optim.AdamW(model.parameters(), lr=1e-2, weight_decay=1e-2)
    else:
        opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    opt = dear.DistributedOptimizer(opt, model, threshold=0.05, verbose=False)
    dear.broadcast_parameters(model.state_dict(), 0)
    step = TrainStep(model, opt, nn.functional.cross_entropy, use_graph=use_graph, graph_warmup=2, overlap_update=overlap)
    g = torch.Generator().manual_seed(100 + rank)
    losses = []
    for t in range(8):
        x = torch.randn(32, 64, generator=g).to(dev)
        y = torch.randint(0, 10, (32,), generator=g).to(dev)
        losses.append(float(step(x, y)))
    opt.synchronize()
    dear.communicator().check_status()
    return losses, [p.detach().float().cpu() for p in model.parameters()], step._graph is not None


@pytest.mark.parametrize("world", [1, 2])
def test_cuda_graph_replay_matches_eager(world):
    eager = run_ranks(graph_worker, world=world, backend="b200", args=(False,), extra_env=_env(), timeout=300)
    graph = run_ranks(graph_worker, world=world, backend="b200", args=(True,), extra_env=_env(), timeout=300)
    assert graph[0][2] and not eager[0][2]
    for (le, pe, _), (lg, pg, _) in zip(eager, graph):
        torch.testing.assert_close(torch.tensor(lg), torch.tensor(le), rtol=1e-4, atol=1e-5)
        for a, b in zip(pg, pe):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2])
def test_rotated_cuda_graph_matches_eager(world):
    """overlap_update: the captured body is step(previous gradients) -> forward -> backward, so the update +
    all-gather kernels are the first nodes of the graph and overlap the forward; same training run."""
    eager = run_ranks(graph_worker, world=world, backend="b200", args=(False,), extra_env=_env(), timeout=300)
    graph = run_ranks(graph_worker, world=world, backend="b200", args=(True, True), extra_env=_env(), timeout=300)
    assert graph[0][2]
    for (le, pe, _), (lg, pg, _) in zip(eager, graph):
        torch.testing.assert_close(torch.tensor(lg), torch.tensor(le), rtol=1e-4, atol=1e-5)
        for a, b in zip(pg, pe):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


def gpu_rebucket_worker(rank, world, steps, per_rank):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    case = dict(momentum=0.9, weight_decay=1e-3)
    model = make_model().to(dev)
    model.eval()
    opt = torch.optim.SGD(model.parameters(), lr=0.05, **case)
    opt = dear.DistributedOptimizer(opt, model, threshold=0.001, verbose=False)
    dear.broadcast_parameters(model.state_dict(), 0)
    layouts = []
    for t in range(steps):
        if t == 2:
            opt.engine.request_rebucket(("threshold", 0.004))
        if t == 4:
            opt.engine.request_rebucket(("nearby", -1))
        x, y = data(t, world * per_rank)
        x, y = x[rank * per_rank:(rank + 1) * per_rank].to(dev), y[rank * per_rank:(rank + 1) * per_rank].to(dev)
        opt.zero_grad()
        nn.functional.cross_entropy(model(x), y).backward()
        opt.step()
        layouts.append(len(opt.engine.plan.buckets))
    opt.synchronize()
    dear.communicator().check_status()
    return [p.detach().float().cpu() for p in model.parameters()], layouts


def test_rebucketing_on_gpu_migrates_sharded_state():
    """dopt_rsag_bo's re-bucketing at the safe point, on the fused path: new symmetric arenas are
    rendezvoused, parameters and the sharded momentum move, training stays equivalent to SGD."""
    case = dict(momentum=0.9, weight_decay=1e-3)
    ref = reference_run(case, 7, 2, 4)
    outs = run_ranks(gpu_rebucket_worker, world=2, backend="b200", args=(7, 4), extra_env=_env(), timeout=300)
    for params, layouts in outs:
        assert len(set(layouts)) == 3 and layouts[-1] == 1
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_adamw_cuda_graph_matches_eager():
    eager = run_ranks(graph_worker, world=2, backend="b200", args=(False, False, True), extra_env=_env(), timeout=300)
    graph = run_ranks(graph_worker, world=2, backend="b200", args=(True, True, True), extra_env=_env(), timeout=300)
    for (le, pe, _), (lg, pg, _) in zip(eager, graph):
        torch.testing.assert_close(torch.tensor(lg), torch.tensor(le), rtol=1e-4, atol=1e-5)
        for a, b in zip(pg, pe):
            torch.testing.assert_close(a, b, rtol=2e-4, atol=2e-5)


def bo_graph_worker(rank, world):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200.utils.train import TrainStep
    dev = dear.device()
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 10)).to(dev)
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
    opt = dear.DistributedOptimizer(opt, model, threshold=0.05, verbose=False, bo_tuning=True,
                                    bo_kwargs=dict(bound=(0.01, 1.0), max_num_steps=3, interval=4))
    dear.broadcast_parameters(model.state_dict(), 0)
    step = TrainStep(model, opt, nn.functional.cross_entropy, use_graph=True, graph_warmup=2)
    g = torch.Generator().manual_seed(100 + rank)
    captured_at = None
    for t in range(40):
        x = torch.randn(32, 64, generator=g).to(dev)
        y = torch.randint(0, 10, (32,), generator=g).to(dev)
        loss = float(step(x, y))
        assert loss == loss
        if captured_at is None and step._graph is not None:
            captured_at = t
            assert opt.tuner.finished
    opt.synchronize()
    dear.communicator().check_status()
    return captured_at, opt.tuner.finished, len(opt.engine.plan.buckets)


@pytest.mark.gpu
def test_graph_capture_waits_for_the_bo_tuner():
    outs = run_ranks(bo_graph_worker, world=2, backend="b200", extra_env=_env(), timeout=300)
    assert outs[0] == outs[1]
    captured_at, finished, _ = outs[0]
    assert finished and captured_at is not None and captured_at >= 12       # 3 trials x 4-iteration windows first


def sched_worker(rank, world, use_graph, overlap):
    """Per-step LR schedule + an eager interruption (state_dict -> finish()) in the middle of graph replays."""
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200.utils.train import TrainStep
    dev = dear.device()
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 10)).to(dev)
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    opt = dear.DistributedOptimizer(opt, model, threshold=0.05, verbose=False)      # several buckets
    dear.broadcast_parameters(model.state_dict(), 0)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.8)            # the LR changes EVERY step
    step = TrainStep(model, opt, nn.functional.cross_entropy, use_graph=use_graph, graph_warmup=2, overlap_update=overlap)
    g = torch.Generator().manual_seed(100 + rank)
    losses = []
    for t in range(12):
        x = torch.randn(32, 64, generator=g).to(dev)
        y = torch.randint(0, 10, (32,), generator=g).to(dev)
        losses.append(float(step(x, y)))
        sched.step()            # the rotated body defers the update of batch t to the start of call t+1, but with the
        #                         hyper-parameters frozen at the end of call t (DearEngine.freeze_hyper): same loop
        if t == 7:
            opt.synchronize()   # rotated: finish() applies the pending update eagerly, then the loop continues
    opt.synchronize()
    dear.communicator().check_status()
    return losses, [p.detach().float().cpu() for p in model.parameters()], step._graph is not None


_SCHED_EAGER = []


def test_cuda_graph_with_lr_scheduler_and_eager_interruption():
    """Advisor finding (round 1): an LR change after capture must not clobber the table a captured kernel reads, and an
    eager step between replays must not leave the graph with the eager step's gradient addresses.  (The rotated body with
    its frozen hyper-parameters: tests/test_zz_post_budget_gpu.py — written after the round's last GPU session.)"""
    check_graph_with_lr_scheduler(False)


def check_graph_with_lr_scheduler(overlap):
    if not _SCHED_EAGER:          # the eager oracle is the same for both parametrisations: run it once
        _SCHED_EAGER.append(run_ranks(sched_worker, world=1, backend="b200", args=(False, False), extra_env=_env(), timeout=300))
    eager = _SCHED_EAGER[0]
    graph = run_ranks(sched_worker, world=1, backend="b200", args=(True, overlap), extra_env=_env(), timeout=300)
    assert graph[0][2]
    (le, pe, _), (lg, pg, _) = eager[0], graph[0]
    # natural and rotated body, replayed or eager: the same losses and the same parameters as the plain eager loop
    # (tests/test_train_step.py checks the rotated loop's schedule semantics against torch on the CPU)
    torch.testing.assert_close(torch.tensor(lg), torch.tensor(le), rtol=1e-4, atol=1e-5)
    for a, b in zip(pg, pe):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


def bcast_bf16_worker(rank, world):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    torch.manual_seed(1000 + rank)                       # every rank starts from DIFFERENT weights
    model = nn.Sequential(nn.Linear(32, 64), nn.ReLU(), nn.Linear(64, 8)).to(dev).to(torch.bfloat16)
    opt = torch.optim.SGD(model.parameters(), lr=0.0)    # lr 0: a step must leave the broadcast values alone
    opt = dear.DistributedOptimizer(opt, model, threshold=0.001, verbose=False)
    dear.broadcast_parameters(model.state_dict(), 0)
    want = [p.detach().float().cpu().clone() for p in model.parameters()]
    x = torch.randn(4, 32, device=dev, dtype=torch.bfloat16)
    model(x).float().sum().backward()
    opt.step()
    opt.synchronize()
    return want, [p.detach().float().cpu() for p in model.parameters()]


def test_broadcast_after_wrapping_updates_the_fp32_masters():
    outs = run_ranks(bcast_bf16_worker, world=2, backend="b200", extra_env=_env(), timeout=300)
    root = outs[0][0]
    for want, got in outs:
        for a, b, r in zip(want, got, root):
            assert torch.equal(a, r), "broadcast did not deliver rank 0's values"
            assert torch.equal(a, b), "an lr=0 step moved the parameters: stale master shards were pushed"


@pytest.mark.parametrize("dtype_name", ["fp32"])     # (bf16 through the pipelined kernel: tests/test_kernels_direct.py)
def test_engine_on_the_pipelined_reduce_scatter(dtype_name):
    """Whole engine (hooks, steal-mode pack tables, sharded update) with every bucket forced onto the stripe-pipelined
    Kernel A (csrc/rs_pipe.cu) and the all-gathers on their own stream."""
    case = dict(momentum=0.9)
    ref = reference_run(case, 3, 2, 4)
    env = dict(_env(), DEAR_RS_ALGO="pipe", DEAR_PIPE_MIN_MB="0", DEAR_STRIPE_MB="0.03125")
    outs = run_ranks(gpu_worker, world=2, backend="b200", args=(case, 3, 4, 0.001, dtype_name), extra_env=env, timeout=300)
    tol = dict(rtol=1e-4, atol=1e-5) if dtype_name == "fp32" else dict(rtol=5e-2, atol=5e-2)
    for params, _ in outs:
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, **tol)
    for a, b in zip(outs[0][0], outs[-1][0]):
        assert torch.equal(a, b)


def test_single_stream_option_still_works():
    case = CASES[2]
    ref = reference_run(case, 3, 2, 2)
    outs = run_ranks(gpu_worker, world=2, backend="b200", args=(case, 3, 2, 0.001, "fp32"),
                     extra_env=dict(_env(), DEAR_AG_STREAM="0"), timeout=300)
    for params, _ in outs:
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
