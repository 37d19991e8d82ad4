"""Cross-GPU migration (needs >= 2 GPUs; skipped on a 1-GPU box): two processes, one per GPU, CUDA-IPC mapped
destination pool, page->page kernel over NVLink; destination pages must equal source pages bit-exact."""
import importlib
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        kvb = importlib.import_module("llm-d-kv-cache_b200")
        part, mig = kvb.partition, kvb.migrate
        T, N, frag, n = 16, 256, 16384, 100
        g = torch.Generator(device="cuda").manual_seed(7 + rank)
        big = torch.randint(0, 256, (T, N, frag), dtype=torch.uint8, device="cuda", generator=g)
        tensors = list(big.unbind(0))
        pool = kvb.pool.KVPool(tensors)
        descs = part.exchange_objects(mig.export_pool(pool), dist)
        dst, src = part.ring_peers(rank, world)
        src_ids = np.random.default_rng(rank).permutation(N // 2)[:n].astype(np.int64)
        dst_ids = (N // 2 + np.random.default_rng(50 + rank).permutation(N // 2)[:n]).astype(np.int64)
        expect = [t[torch.from_numpy(src_ids).cuda()].cpu() for t in tensors]
        untouched = [t[: N // 2].clone() for t in tensors]
        remote = mig.RemotePool(descs[dst], rank)
        for variant in (1, 2):
            mig.migrate_blocks(pool, remote, src_ids, dst_ids, flags=variant)
            torch.cuda.synchronize()
            dist.barrier()
            # ship what I sent to the rank that received it and compare there
            meta = part.exchange_objects({"ids": dst_ids.tolist(), "pages": [e.numpy() for e in expect]}, dist)
            got_ids = torch.tensor(meta[src]["ids"], device="cuda")
            for t, want in zip(tensors, meta[src]["pages"]):
                assert np.array_equal(t[got_ids].cpu().numpy(), want)
            for t, u in zip(tensors, untouched):
                assert torch.equal(t[: N // 2], u)          # lower half (source pages) never written
            for t in tensors:
                t[N // 2:] = 0
            torch.cuda.synchronize()
            dist.barrier()
        remote.close()
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_ring_migration_two_gpus(torch_cuda):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert res == {0: "ok", 1: "ok"}, res
