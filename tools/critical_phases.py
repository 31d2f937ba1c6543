"""Where the critical block's time goes: one C2 compression (the call bench.py times: 100 MB of text,
gzip, numiterations=15, input resident on the device), then the six k_iterate phase counters of the
block with the largest cycle total, as SM cycles per position-iteration, with the card, its power limit
and the SM clock sampled during the call.

usage: python tools/critical_phases.py [--warmup W] [--runs R]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["model", "dp", "trace", "follow", "block_size", "statistics"]   # JobState::cyc (kernels.cuh)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--runs", type=int, default=1)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import zopfli_b200 as zb

    torch.cuda.set_device(0)
    lib = zb.library()
    data, kind = bench.workload(bench.SHARD, 2)
    host = np.zeros(len(data) + 64, dtype=np.uint8)
    host[:len(data)] = np.frombuffer(data, dtype=np.uint8)
    dev = torch.zeros(len(host), dtype=torch.uint8, device="cuda")
    dev[:len(data)].copy_(torch.from_numpy(host[:len(data)]))
    torch.cuda.synchronize()

    def job():
        lib.compress_ptr_nocopy(host.ctypes.data, len(data), zb.ZOPFLI_FORMAT_GZIP, dev_ptr=dev.data_ptr(),
                                numiterations=bench.NUMITER).close()

    for _ in range(args.warmup):
        job()
    for _ in range(args.runs):
        lib.reset_stats()
        sampler = bench.ClockSampler(0)
        sampler.start()
        job()
        sampler.stop_flag = True
        sampler.join()
        st = lib.stats()
        cyc = st["cyc_max"]
        steps = max(1, int(st["max_block_positions"]) * bench.NUMITER)
        per = {p: c / steps for p, c in zip(PHASES, cyc)}
        clocks = sampler.summary()
        print(json.dumps({"data": kind, "max_block_positions": int(st["max_block_positions"]),
                          "iterations": bench.NUMITER, "cycles_per_step": per,
                          "all_cycles_per_step": sum(cyc) / steps,
                          "non_dp_cycles_per_step": (sum(cyc) - cyc[1]) / steps,
                          "gpu": clocks["gpu"], "power_limit_w": clocks["power_limit_w"],
                          "sm_mhz": clocks["sm_mhz"], "sm_max_mhz": clocks["sm_max_mhz"],
                          "throttle_reasons": clocks["reasons"]}), flush=True)


if __name__ == "__main__":
    main()
