"""Two-process GPU tests of the data-parallel path that bench.py / SCALE measure: one process per GPU, weights
replicated, batch sharded by parallel.shard_bounds, decoded shards all-gathered by the library over NVLink peer memory
(north_star: "one all-gather of decoded images and nothing else").

Covered, each against the locally recomputed full batch (every rank can reconstruct every shard: same weights):
  * fused form   (ian_reconstruct_gather_dev): dec_out stores straight into every rank's buffer + flag barrier
  * pipelined form (ian_reconstruct_gather_async_dev / ian_gather_wait_dev): side-stream push (copy engines + stream
    memory operations by default; IAN_PUSH=kernel: the copy kernel) + free/pushed flags
  * shards larger than the 512-image plan chunk
  * RANK SKEW: one rank is delayed by a long device-side sleep before some steps, so a rank that runs ahead would
    overwrite a buffer its peer is still reading if the lifetime contract of include/ian_b200.h did not hold
  * IAN.reconstruct_sharded, the public entry that goes through parallel.shard_bounds

Needs >= 2 GPUs: skipped on a machine with one GPU; run with `python -m pytest tests/test_gpu_multi.py` on two or more.
"""
import importlib
import os
import socket
import sys
import traceback

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    try:
        if ROOT not in sys.path:
            sys.path.insert(0, ROOT)
        import torch
        import torch.distributed as dist
        from oracle import weights as ow
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        pkg = importlib.import_module("neural-photo-editor_b200")
        par = importlib.import_module("neural-photo-editor_b200.parallel")
        model = pkg.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0), device=rank)
        stream = torch.cuda.Stream(device=dev)
        torch.cuda.set_stream(stream)
        res = {}

        def run_case(tag, n_local, steps, pipelined):
            n = n_local * world
            lo, hi = par.shard_bounds(n, rank, world)
            model.setup_fused_gather(n_local) if not hasattr(model, "_gather_n") else None
            worst = 0.0
            for t in range(steps):
                x = torch.from_numpy(np.random.default_rng(100 * t + 7).uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).to(dev)
                want = torch.empty_like(x)
                model.reconstruct_dev(x.data_ptr(), n, 0, want.data_ptr(), stream.cuda_stream)      # the full batch, locally
                if (t + rank) % 2 == 0:
                    torch.cuda._sleep(int(4e8))                   # ~0.2 s of device-side delay on alternating ranks
                shard = x[lo:hi].contiguous()
                if pipelined:
                    model.reconstruct_gather_async_dev(shard.data_ptr(), n_local, 0, stream.cuda_stream)
                    ptr = model.gather_wait_dev(stream.cuda_stream)
                else:
                    ptr = model.reconstruct_gather_dev(shard.data_ptr(), n_local, 0, stream.cuda_stream)
                got = par.as_cuda_tensor(ptr, (n, 3, 64, 64), dev)
                err = (got - want).abs().max()                    # consumer enqueued in stream order BEFORE the next call
                if (t + rank) % 2 == 1:
                    torch.cuda._sleep(int(2e8))                   # ... and the slow consumer side of the skew
                worst = max(worst, float(err.item()))
            res[tag] = worst

        run_case("fused", 6, 6, False)
        run_case("pipelined", 6, 6, True)                 # copy engines + stream memory operations (default push)
        run_case("mixed", 6, 4, False)
        model.close()
        os.environ["IAN_PUSH"] = "kernel"                 # the copy-KERNEL form of the push (read when the side stream is made)
        model = pkg.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0), device=rank)
        run_case("pipelined_push_kernel", 6, 6, True)
        model.close()
        del os.environ["IAN_PUSH"]
        # shards above the 512-image plan chunk, both forms, through the public sharded entry
        model = pkg.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0), device=rank)
        n = 2 * 520
        x = torch.from_numpy(np.random.default_rng(5).uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).to(dev)
        want = torch.empty_like(x)
        model.reconstruct_dev(x.data_ptr(), n, 0, want.data_ptr(), stream.cuda_stream)
        for tag, pip in (("sharded_fused_520", False), ("sharded_pipelined_520", True)):
            got = model.reconstruct_sharded(x, stream=stream.cuda_stream, pipelined=pip)
            res[tag] = float((got - want).abs().max().item())
        torch.cuda.synchronize()
        model.close()
        dist.destroy_process_group()
        q.put((rank, res, None))
    except Exception:
        q.put((rank, None, traceback.format_exc()))


def test_two_gpu_gather_fused_pipelined_chunked_with_rank_skew():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    for rank, res, err in out:
        assert err is None, "rank %d:\n%s" % (rank, err)
        # batch-size dependent split-K factors: a shard run alone vs inside the full batch differs like two float32
        # summation orders (tests/test_gpu_parity.py: X_RERUN)
        for tag, v in res.items():
            assert v <= 5e-5, (rank, tag, v)
    if os.environ.get("IAN_TEST_RECORD"):
        import json
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "two_gpu_gather.json"), "w") as f:
            json.dump({str(r): res for r, res, _ in out}, f)
