"""Device-resident compression and device checksums, measured in one run on one GPU.

C2 (bench.py's workload: 100,000,000 bytes of synthetic text, gzip, numiterations=15, input resident in
HBM), alternating
  (a) ZopfliB200CompressDevice          -- device input, result in host memory, CRC-32 on the host
  (b) ZopfliB200CompressDeviceToDevice  -- device input, result in device memory, CRC-32 on the device
with the bytes of (a) and (b) compared.  Then CRC-32 and Adler-32 of the same 100 MB on the device: the
time per blocking call from CUDA events over many calls, and the kernels' own time from torch.profiler,
as GB/s and as a fraction of the HBM peak; and the threaded host CRC-32 (ZopfliB200Crc32) for comparison.
Prints one JSON line per measurement, each with the card's name and power limit.

usage: python tools/device_resident_bench.py [--warmup W] [--runs R] [--launches L]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    o = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(",")
    return {"gpu": o[0].strip(), "power_limit_w": float(o[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import zopfli_b200 as zb

    torch.cuda.set_device(0)
    lib = zb.library()
    info = card()
    data, kind = bench.workload(bench.SHARD, 2)
    n = len(data)
    host = np.zeros(n + 64, dtype=np.uint8)
    host[:n] = np.frombuffer(data, dtype=np.uint8)
    dev = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    dev[:n].copy_(torch.from_numpy(host[:n]))
    x = dev[:n]
    torch.cuda.synchronize()

    def leg_a():
        ob = lib.compress_ptr_nocopy(host.ctypes.data, n, zb.ZOPFLI_FORMAT_GZIP, dev_ptr=dev.data_ptr(),
                                     numiterations=bench.NUMITER)
        b = ob.tobytes()
        ob.close()
        return b

    def leg_b():
        out = lib.compress_device(x, zb.ZOPFLI_FORMAT_GZIP, numiterations=bench.NUMITER)
        return out

    legs = {"a_compress_device": leg_a, "b_compress_device_to_device": leg_b}
    for _ in range(args.warmup):
        for f in legs.values():
            f()
    ms = {k: [] for k in legs}
    outs = {}
    for _ in range(args.runs):
        for k, f in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = f()
            ms[k].append((time.perf_counter() - t0) * 1e3)  # both calls return after a device synchronise
            outs[k] = r
    same = outs["a_compress_device"] == bytes(outs["b_compress_device_to_device"].cpu().numpy())
    for k in legs:
        med = statistics.median(ms[k])
        print(json.dumps({"leg": k, "data": kind, "bytes": n, "out_bytes": len(outs[k]), "ms_per_call": ms[k],
                          "median_ms": med, "median_mib_s": n / (1 << 20) / (med / 1e3), **info}), flush=True)
    print(json.dumps({"identical_bytes": bool(same), **info}), flush=True)
    del outs

    peak, peak_src = bench.peak_hbm()  # GB/s
    for name, fn, ref in (("crc32", lib.crc32_device, lambda: lib.crc32(host.ctypes.data, n)),
                          ("adler32", lib.adler32_device, None)):
        for _ in range(5):
            fn(x)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            fn(x)
        e1.record()
        e1.synchronize()
        call_ms = e0.elapsed_time(e1) / args.launches
        kern_ms = None
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                fn(x)
            torch.cuda.synchronize()
        ks = [e for e in prof.key_averages() if ("k_" + name) in e.key]
        if ks and ks[0].count:
            total_us = getattr(ks[0], "device_time_total", None) or getattr(ks[0], "cuda_time_total", 0)
            kern_ms = total_us / ks[0].count / 1e3
        rec = {"checksum": name, "bytes": n, "value": fn(x), "zlib_check": None,
               "call_ms": call_ms, "call_gb_s": n / call_ms / 1e6, "call_fraction_of_peak": n / call_ms / 1e6 / peak,
               "kernel_ms": kern_ms, "kernel_gb_s": n / kern_ms / 1e6 if kern_ms else None,
               "kernel_fraction_of_peak": n / kern_ms / 1e6 / peak if kern_ms else None,
               "hbm_peak_gb_s": peak, "hbm_peak_source": peak_src, **info}
        import zlib
        rec["zlib_check"] = rec["value"] == (zlib.crc32(data) if name == "crc32" else zlib.adler32(data))
        if ref:
            t0 = time.perf_counter()
            reps = 5
            for _ in range(reps):
                ref()
            host_ms = (time.perf_counter() - t0) * 1e3 / reps
            rec.update(host_crc32_ms=host_ms, host_crc32_gb_s=n / host_ms / 1e6)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
