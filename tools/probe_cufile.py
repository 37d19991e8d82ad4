#!/usr/bin/env python
"""Is GPUDirect Storage usable on this box?  Reports the nvidia-fs kernel module, what cuFileDriverOpen returns, and
whether cuFileHandleRegister / cuFileWrite / cuFileRead work from device memory on a few file systems
(without the module the driver opens in compatibility mode, see csrc/engine.cu)."""
import ctypes
import os
import subprocess

import torch

print("nvidia_fs module:", subprocess.run("lsmod | grep -i nvidia_fs; ls /proc/driver/nvidia-fs 2>&1 | head -2", shell=True,
                                          capture_output=True, text=True).stdout.strip() or "absent")


class Err(ctypes.Structure):
    _fields_ = [("err", ctypes.c_int), ("cu_err", ctypes.c_int)]


class Descr(ctypes.Structure):  # CUfileDescr_t: type, handle union (fd / void*), fs_ops*
    _fields_ = [("type", ctypes.c_int), ("fd", ctypes.c_int64), ("fs_ops", ctypes.c_void_p)]


lib = ctypes.CDLL("/usr/local/cuda/lib64/libcufile.so")
lib.cuFileDriverOpen.restype = Err
lib.cuFileHandleRegister.restype = Err
lib.cuFileHandleRegister.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(Descr)]
lib.cuFileWrite.restype = ctypes.c_ssize_t
lib.cuFileWrite.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int64]
lib.cuFileRead.restype = ctypes.c_ssize_t
lib.cuFileRead.argtypes = lib.cuFileWrite.argtypes
lib.cuFileHandleDeregister.argtypes = [ctypes.c_void_p]
torch.zeros(1, device="cuda")
r = lib.cuFileDriverOpen()
print("cuFileDriverOpen ->", r.err, r.cu_err)
src = torch.arange(1 << 20, dtype=torch.uint8, device="cuda")
dst = torch.zeros_like(src)
for d in ("/tmp", "/dev/shm", "/root", "/var/tmp"):
    for direct in (True, False):
        path = os.path.join(d, "kvb_cufile_probe.bin")
        try:
            fd = os.open(path, os.O_RDWR | os.O_CREAT | os.O_TRUNC | (os.O_DIRECT if direct else 0), 0o644)
        except OSError as e:
            print(f"{d:9s} O_DIRECT={direct}: open failed: {e}")
            continue
        h = ctypes.c_void_p()
        desc = Descr(1, fd, None)
        st = lib.cuFileHandleRegister(ctypes.byref(h), ctypes.byref(desc))
        msg = f"{d:9s} O_DIRECT={direct}: register err={st.err}"
        if st.err == 0:
            w = lib.cuFileWrite(h, src.data_ptr(), src.numel(), 0, 0)
            rd = lib.cuFileRead(h, dst.data_ptr(), dst.numel(), 0, 0)
            torch.cuda.synchronize()
            msg += f" write={w} read={rd} equal={bool(torch.equal(src, dst))}"
            lib.cuFileHandleDeregister(h)
        os.close(fd)
        os.unlink(path)
        print(msg, flush=True)
        dst.zero_()
print(subprocess.run("df -T /tmp /dev/shm /root 2>/dev/null | awk '{print $1, $2, $7}'", shell=True, capture_output=True, text=True).stdout)
