"""Time the matrix-file writer (mb_save_rows / mb_save_blocks behind saveToFileSystem) against the host writer it replaces.

Workloads: a 1048576 x 1024 uniform [0, 1) row shard and a 16384 x 16384 BlockMatrix in 2 x 2 blocks.  For each:
  * kernels alone: the durations of text_length_kernel and text_write_kernel, and of the device-to-host copies, summed
    from a torch.profiler trace of one save to /dev/null (a run of its own);
  * end to end without a file system: host clock around one save to /dev/null (kernels, copies, pipeline);
  * end to end: host clock around saveToFileSystem into a temporary directory, when the file system has room for it;
    the file-write share is this minus the /dev/null time;
  * the host writer (_jdouble per value): timed on a 2^20-value sample and extrapolated, labelled as such.
Text bytes per workload are the size of the file written (or, without room for it, estimated from the first 2^21 values'
file and labelled so).  The card's name and power limit are read in the same run.  Prints one JSON line per workload.

    python scripts/bench_text.py [--workloads rows,blocks] [--tmp DIR]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import _native as nat
from marlin_b200.utils.mt_utils import _jdouble


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def save(rt, target, path):
    """One blocking save of target (a DenseVecMatrix or [(rc, SubMatrix)]) to path through the C ABI; seconds."""
    rt.sync_stream()
    torch.cuda.synchronize()
    t = time.perf_counter()
    if isinstance(target, mb.DenseVecMatrix):
        ids = np.ascontiguousarray(target.ids, dtype=np.int64)
        nat.check(rt.lib.mb_save_rows(rt.ctx, target.data.handle(), ids.ctypes.data_as(C.c_void_p), os.fsencode(path)))
    else:
        handles = (nat.c_blk * len(target))(*[s.handle() for _, s in target])
        rc = np.array([list(k) for k, _ in target], dtype=np.int32).reshape(-1)
        nat.check(rt.lib.mb_save_blocks(rt.ctx, handles, rc.ctypes.data_as(C.c_void_p), len(target), os.fsencode(path)))
    return time.perf_counter() - t


def profile(rt, target):
    """(format kernel seconds, device-to-host copy seconds) of one save to /dev/null."""
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        save(rt, target, "/dev/null")
        torch.cuda.synchronize()
    kern = copy = 0.0
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "text_length_kernel" in e.name or "text_write_kernel" in e.name:
            kern += us * 1e-6
        elif "DtoH" in e.name or "Device -> Pageable" in e.name or "Device -> Pinned" in e.name:
            copy += us * 1e-6
    return kern, copy


def host_writer_per_value(sample):
    t = time.perf_counter()
    ",".join(_jdouble(v) for v in sample)
    return (time.perf_counter() - t) / len(sample)


def workload(name, tmp):
    rt = mb.Runtime.get()
    dev = rt.device
    g = torch.Generator(device=dev).manual_seed(20261018)
    if name == "rows":
        rows, cols = 1048576, 1024
        data = mb.SubMatrix(buf=torch.rand(rows * cols, dtype=torch.float64, device=dev, generator=g), rows=rows, cols=cols,
                            ld=cols, is_transpose=True)
        target = mb.DenseVecMatrix(ids=np.arange(rows), data=data, nRows=rows, nCols=cols)
        head = mb.DenseVecMatrix(ids=np.arange(2048), data=data.slice(0, 2048, 0, cols), nRows=rows, nCols=cols)
        n = rows * cols
    else:
        side, half = 16384, 8192
        target = [((r, c), mb.SubMatrix(buf=torch.rand(half * half, dtype=torch.float64, device=dev, generator=g), rows=half,
                                         cols=half, ld=half)) for r in range(2) for c in range(2)]
        head = [((0, 0), target[0][1].slice(0, half, 0, 256))]
        n = side * side
    d = tempfile.mkdtemp(dir=tmp)
    try:
        save(rt, head, os.path.join(d, "head"))                                     # warm-up; the sample's text
        per_value = os.path.getsize(os.path.join(d, "head")) / (2048 * 1024 if name == "rows" else half * 256)
        os.remove(os.path.join(d, "head"))
        est_bytes = per_value * n
        devnull = min(save(rt, target, "/dev/null") for _ in range(2))
        kern, copy = profile(rt, target)
        res = {"workload": name, "values": n, **card(), "devnull_s": devnull, "kernel_s": kern, "d2h_s": copy}
        free = shutil.disk_usage(d).free
        if free > 1.2 * est_bytes:
            part = os.path.join(d, "part-00000")
            e2e = save(rt, target, part)
            res.update(bytes=os.path.getsize(part), bytes_measured=True, e2e_s=e2e, file_write_s=e2e - devnull)
            os.remove(part)
        else:
            res.update(bytes=int(est_bytes), bytes_measured=False, e2e_s=None,
                       e2e_note=f"not measured: {free / 1e9:.1f} GB free in {tmp}, about {est_bytes / 1e9:.1f} GB needed")
        res["kernel_values_per_s"] = n / kern if kern else None
        res["kernel_text_GBps"] = res["bytes"] / kern / 1e9 if kern else None
        res["d2h_GBps"] = res["bytes"] / copy / 1e9 if copy else None
        res["devnull_GBps"] = res["bytes"] / devnull / 1e9
        if res.get("e2e_s"):
            res["e2e_GBps"] = res["bytes"] / res["e2e_s"] / 1e9
        sample = np.random.default_rng(1).random(1 << 20)
        res["host_writer_s_per_value"] = host_writer_per_value(sample)
        res["host_writer_s_extrapolated"] = res["host_writer_s_per_value"] * n
        return res
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="rows,blocks")
    ap.add_argument("--tmp", default=tempfile.gettempdir())
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text.py needs a CUDA device")
    for w in a.workloads.split(","):
        print(json.dumps(workload(w, a.tmp)), flush=True)


if __name__ == "__main__":
    main()
