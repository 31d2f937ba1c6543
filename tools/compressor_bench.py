"""Input in pieces against the whole buffer: ZopfliCompress of one input, and ZopfliB200Compressor fed the same
bytes in 1 MiB and 64 MiB writes from host memory and from device memory, alternating in one process.

The input is C2's text (corpus.synth_text, seed 2) at --mib MiB; the default, 430 MiB, is six waves and a
part of an 80 GB card (a wave is 72 master blocks there).  Every run prints one JSON line with its time and
rate, and the device memory in use after it (cudaMemGetInfo), so that growth across repetitions shows; every
compressor output is checked against ZopfliCompress's.  The card's name, power limit and clock limit are read
in the same run.

With --flush-every BYTES, two more legs (host and device chunks, 64 MiB writes) end a sync flush every BYTES of
input: each flush runs what has arrived as a wave of its own, however short.  Their output differs from
ZopfliCompress's by the flush points, so it is checked by inflating it instead.

With --restart-every BYTES, two more legs (host chunks, 64 MiB writes) put a full flush every BYTES of input: one
calls Flush(FULL) at each point, so each point ends a wave of its own; the other sets restart_interval=BYTES, so
the segments between points share waves.  Their streams must be byte-identical ("identical_to_explicit"), and
every index entry of the restart leg must inflate raw to the data from its offset on.

With --device-output, one more leg (device chunks, 64 MiB writes) takes its output in device memory
(compressobj(..., device_output=True)); its stream must be byte-identical to the device-chunk leg's with host
output ("identical_to_host_output").  Every record then also carries the leg's h2d_bytes and d2h_bytes
(ZopfliB200Stats), which show what crossed PCIe.

    python tools/compressor_bench.py [--mib 430] [--reps 3] [--numiterations 15] [--flush-every BYTES]
                                     [--restart-every BYTES] [--device-output]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import zlib

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


def run_pieces(lib, src, write, kw, device, flush_every=0, mode=zlib.Z_SYNC_FLUSH, restart_interval=None,
               index=None, device_output=False):
    out = []
    with lib.compressobj(zb.ZOPFLI_FORMAT_GZIP, device=0 if device else None, restart_interval=restart_interval,
                         device_output=device_output, **kw) as c:
        p = 0
        while p < len(src):
            q = min(p + write, len(src))
            if flush_every:
                q = min(q, (p // flush_every + 1) * flush_every)
            out.append(c.compress(src[p:q]))
            p = q
            # a full flush only where data follows, as restart points are placed
            if flush_every and p % flush_every == 0 and (mode == zlib.Z_SYNC_FLUSH or p < len(src)):
                out.append(c.flush(mode))
        out.append(c.flush())
        if index is not None:
            index[:] = c.restart_points()
    return torch.cat(out) if device_output else b"".join(out)


def index_inflates(stream, data, index):
    """every entry's first 64 KiB inflate raw to the data from its offset on"""
    return all(zlib.decompressobj(-15).decompress(stream[s:], 65536) == data[d:d + 65536] for d, s in index)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=430)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--numiterations", type=int, default=15)
    ap.add_argument("--flush-every", type=int, default=0, help="bytes of input between sync flushes (0: no flush legs)")
    ap.add_argument("--restart-every", type=int, default=0,
                    help="bytes of input between full flushes, explicit and by restart_interval (0: no restart legs)")
    ap.add_argument("--device-output", action="store_true",
                    help="a leg with device chunks and output in device memory, and PCIe bytes in every record")
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
    f = args.flush_every
    if f:
        legs.append(("compressor host 64 MiB, sync flush every %d B" % f,
                     lambda: run_pieces(lib, host_view, 64 * MIB, kw, False, f)))
        legs.append(("compressor device 64 MiB, sync flush every %d B" % f,
                     lambda: run_pieces(lib, dev, 64 * MIB, kw, True, f)))
    r = args.restart_every
    index = []
    if r:
        legs.append(("compressor host 64 MiB, Flush(FULL) every %d B" % r,
                     lambda: run_pieces(lib, host_view, 64 * MIB, kw, False, r, zlib.Z_FULL_FLUSH)))
        legs.append(("compressor host 64 MiB, restart_interval=%d" % r,
                     lambda: run_pieces(lib, host_view, 64 * MIB, kw, False, restart_interval=r, index=index)))
    if args.device_output:
        legs.append(("compressor device 64 MiB, device output",
                     lambda: run_pieces(lib, dev, 64 * MIB, kw, True, device_output=True)))
    want, explicit, device_host_output = None, None, None
    for rep in range(args.reps):
        for name, fn in legs:
            torch.cuda.synchronize()
            lib.reset_stats()
            t0 = time.perf_counter()
            got = fn()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            st = lib.stats()
            if isinstance(got, torch.Tensor):  # device output: copied to the host for the checks, after the timing
                got = bytes(got.cpu().numpy())
            if want is None:
                want = got
            free, total = torch.cuda.mem_get_info(0)
            rec = {"rep": rep, "leg": name, "ms": round(ms, 1), "MiB_s": round(len(data) / MIB / (ms / 1e3), 2),
                   "out_bytes": len(got)}
            if "Flush(FULL)" in name:
                explicit = got
                rec["inflates"] = zlib.decompress(got, 31) == data
            elif "restart_interval" in name:
                rec["identical_to_explicit"] = got == explicit
                rec["restart_points"] = len(index)
                rec["index_inflates"] = index_inflates(got, data, index)
            elif "flush" in name:
                rec["inflates"] = zlib.decompress(got, 31) == data
            else:
                rec["identical"] = got == want
            if name == "compressor device 64 MiB":
                device_host_output = got
            elif "device output" in name:
                rec["identical_to_host_output"] = got == device_host_output
            if args.device_output:
                rec["h2d_bytes"], rec["d2h_bytes"] = st["h2d_bytes"], st["d2h_bytes"]
            rec["device_used_GiB"] = round((total - free) / (1 << 30), 2)
            print(json.dumps(rec), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
