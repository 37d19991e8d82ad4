"""Interop with the unmodified reference engine, pinned by the bytes it wrote.  tests/golden/ref_offload_files.json
holds, per file the reference engine (kv_connectors/llmd_fs_backend, built by oracle/ref_build) stored for the inputs
below, its size, the payload's offset and the SHA-256 of the payload; tests/golden/make_ref_offload_golden.py recorded
them.  Our files must carry the same bytes, and files laid out as the reference writes them must load back through our
engine.  This is what pins oracle/offload_oracle.py (the
reference's own tests hold no golden bytes for this path)."""
import hashlib
import json
import os
import shutil
import time

import numpy as np
import pytest

from oracle import offload_oracle as oo

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TMP = "/tmp/kvb-ref-interop"


def cpu_case(bpf):
    """Inputs of the CPU-path case: T tensors of (N, frag) bytes and three files, the first one partial."""
    T, N, frag = 6, 48, 8192
    rng = np.random.default_rng(11)
    src = [rng.integers(0, 256, (N, frag), dtype=np.uint8) for _ in range(T)]
    ids = [[5, 9][:bpf] if bpf > 1 else [5], list(range(10, 10 + bpf)), list(range(30, 30 + bpf))]
    ids[0] = ids[0][: max(1, bpf // 2)]
    return src, ids


def _drain(eng, job):
    t0 = time.time()
    while time.time() - t0 < 30:
        for j, ok in eng.get_finished():
            if j == job:
                return ok
        time.sleep(0.001)
    raise TimeoutError(job)


def _device(torch, np_src):
    return [torch.from_numpy(a).view(torch.int8).cuda() for a in np_src]


def _loads_back(kvb, torch, src, bpf, files, ids):
    dst = [torch.zeros_like(t) for t in src]
    eng = kvb.engine.StorageOffloadEngine(2, bpf, dst, 1, "disabled", 0.0)
    assert eng.async_load_gpu_blocks(2, files, ids)
    assert _drain(eng, 2)
    torch.cuda.synchronize()
    for blk in ids:
        for d, s in zip(dst, src):
            assert torch.equal(d[blk], s[blk])
    eng.shutdown()


@pytest.mark.parametrize("bpf", [1, 4])
def test_files_interoperate_and_match_oracle(kvb, torch_cuda, bpf):
    torch = torch_cuda
    shutil.rmtree(TMP, ignore_errors=True)
    np_src, ids = cpu_case(bpf)
    T, frag = len(np_src), np_src[0].shape[1]
    src = _device(torch, np_src)
    with open(os.path.join(GOLDEN, "ref_offload_files.json")) as fh:
        gold = json.load(fh)[f"bpf{bpf}"]
    ours = kvb.engine.StorageOffloadEngine(4, bpf, src, 3, "disabled", 0.0)
    f_our = [f"{TMP}/ours/{i}.bin" for i in range(3)]
    assert ours.async_store_gpu_blocks(1, f_our, ids)
    assert _drain(ours, 1)
    ours.shutdown()
    os.makedirs(f"{TMP}/ref")
    f_ref = [f"{TMP}/ref/{i}.bin" for i in range(3)]
    assert len(gold) == len(ids)
    for ref, fo, fr, blk in zip(gold, f_our, f_ref, ids):
        b = np.fromfile(fo, dtype=np.uint8)
        want = oo.file_image(np_src, blk, bpf)
        off, n = oo.slot_offset(T, frag, bpf, len(blk)), len(blk) * T * frag
        assert ref["size"] == b.size == want.size == oo.staging_size(T, frag, bpf)
        assert ref["offset"] == off and ref["payload_bytes"] == n
        # payload region identical in all three; outside it the reference holds stale staging bytes, we hold zeros
        assert hashlib.sha256(b[off:off + n].tobytes()).hexdigest() == ref["payload_sha256"] and np.array_equal(b, want)
        img = np.full(b.size, 0xA5, dtype=np.uint8)       # the reference's file: its payload amid stale bytes
        img[off:off + n] = b[off:off + n]
        img.tofile(fr)
    # files as either implementation wrote them load back into zeroed caches
    for files in (f_ref, f_our):
        _loads_back(kvb, torch, src, bpf, files, ids)
    shutil.rmtree(TMP, ignore_errors=True)
