"""Input in pieces against the whole buffer: ZopfliCompress of one input, and ZopfliB200Compressor fed the same
bytes in 1 MiB and 64 MiB writes from host memory and from device memory, alternating in one process.

The input is C2's text (corpus.synth_text, seed 2) at --mib MiB; the default, 430 MiB, is six waves and a
part of an 80 GB card (a wave is 72 master blocks there).  Every run prints one JSON line with its time and
rate, and the device memory in use after it (cudaMemGetInfo), so that growth across repetitions shows; every
compressor output is checked against ZopfliCompress's.  The card's name, power limit and clock limit are read
in the same run.

    python tools/compressor_bench.py [--mib 430] [--reps 3] [--numiterations 15]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import zopfli_b200 as zb  # noqa: E402
from zopfli_b200 import corpus  # noqa: E402

MIB = 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def run_whole(lib, data, kw):
    a = np.frombuffer(data, np.uint8)
    return lib.compress_ptr(a.ctypes.data, len(data), zb.ZOPFLI_FORMAT_GZIP, **kw)


def run_pieces(lib, src, write, kw, device):
    out = []
    with lib.compressobj(zb.ZOPFLI_FORMAT_GZIP, device=0 if device else None, **kw) as c:
        for p in range(0, len(src), write):
            out.append(c.compress(src[p:p + write]))
        out.append(c.flush())
    return b"".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=430)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--numiterations", type=int, default=15)
    args = ap.parse_args()
    kw = {"numiterations": args.numiterations}
    lib = zb.library()
    t = time.time()
    data = corpus.synth_text(args.mib * MIB, 2)
    dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda:0")
    torch.cuda.synchronize()
    print(json.dumps({"card": card(), "input_bytes": len(data), "input_build_s": round(time.time() - t, 1)}), flush=True)
    host_view = memoryview(data)
    legs = [("ZopfliCompress", lambda: run_whole(lib, data, kw))]
    for write in (1, 64):
        legs.append(("compressor host %d MiB" % write, lambda w=write: run_pieces(lib, host_view, w * MIB, kw, False)))
    for write in (1, 64):
        legs.append(("compressor device %d MiB" % write, lambda w=write: run_pieces(lib, dev, w * MIB, kw, True)))
    want = None
    for rep in range(args.reps):
        for name, fn in legs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = fn()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            if want is None:
                want = got
            free, total = torch.cuda.mem_get_info(0)
            print(json.dumps({"rep": rep, "leg": name, "ms": round(ms, 1), "MiB_s": round(len(data) / MIB / (ms / 1e3), 2),
                              "out_bytes": len(got), "identical": got == want,
                              "device_used_GiB": round((total - free) / (1 << 30), 2)}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
