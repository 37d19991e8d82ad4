#!/usr/bin/env python
"""Record the files the unmodified reference engine writes for the cases of tests/test_gpu_ref_interop.py.

Needs a GPU and the reference engine built into oracle/_ref (oracle/ref_build/build_ref.py):

    python -m tests.golden.make_ref_offload_golden [OUT_DIR]      # default: tests/golden

Writes ref_offload_files.json: per file, its size, the payload's offset and length and the SHA-256 of the payload
region (outside it the reference's files hold stale staging bytes).  Nothing of the reference's code is stored.
"""
import hashlib
import importlib.util
import json
import os
import shutil
import sys
import time

import numpy as np
import torch

from oracle import offload_oracle as oo
from tests.test_gpu_ref_interop import cpu_case

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _drain(eng, job, timeout=30):
    t0 = time.time()
    while time.time() - t0 < timeout:
        for j, ok in eng.get_finished():
            if j == job:
                return ok
        time.sleep(0.001)
    return False


def main(out_dir):
    so = os.path.join(ROOT, "oracle", "_ref", "storage_offload_ref.so")
    spec = importlib.util.spec_from_file_location("storage_offload_ref", so)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    os.makedirs(out_dir, exist_ok=True)
    tmp = "/tmp/kvb-ref-golden"
    golden = {}
    for bpf in (1, 4):
        shutil.rmtree(tmp, ignore_errors=True)
        np_src, ids = cpu_case(bpf)
        T, frag = len(np_src), np_src[0].shape[1]
        src = [torch.from_numpy(a).view(torch.int8).cuda() for a in np_src]
        eng = ref.StorageOffloadEngine(4, bpf, src, 3, "disabled", 0.0)
        files = [f"{tmp}/{i}.bin" for i in range(len(ids))]
        eng.async_store_gpu_blocks(1, files, ids)
        assert _drain(eng, 1), "reference store failed"
        del eng
        golden[f"bpf{bpf}"] = []
        for i, (f, blk) in enumerate(zip(files, ids)):
            img = np.fromfile(f, dtype=np.uint8)
            off, n = oo.slot_offset(T, frag, bpf, len(blk)), len(blk) * T * frag
            golden[f"bpf{bpf}"].append({"size": int(img.size), "offset": off, "payload_bytes": n,
                                        "payload_sha256": hashlib.sha256(img[off:off + n].tobytes()).hexdigest()})
            print(f"bpf={bpf} file {i}: {img.size} bytes, payload equals the oracle:",
                  np.array_equal(img[off:off + n], oo.pack_blocks(np_src, blk)))
    with open(os.path.join(out_dir, "ref_offload_files.json"), "w") as fh:
        json.dump(golden, fh, indent=1)
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
