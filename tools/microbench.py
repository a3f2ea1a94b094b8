#!/usr/bin/env python3
"""Latency / throughput probes of the device arithmetic (zk_debug_op_throughput): how many Montgomery multiplications
(and XYZZ mixed additions) per second the H100 sustains as a function of resident warps and per-thread ILP.
The result is the compute roof DESIGN.md quotes next to the HBM roof."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import proof_systems_b200 as zk

ctx = zk.Context(0)
SMS = torch.cuda.get_device_properties(0).multi_processor_count
CLOCK_HZ = 1.98e9                               # H100 SXM maximum SM clock (nvidia-smi clocks.max.sm)
rows = []
KINDS = ((1, "fe_mul ilp1"), (2, "fe_mul ilp2"), (4, "fe_mul ilp4"), (100, "xyzz_madd"), (102, "xyzz_add"), (101, "xyzz_add_quad"))
if len(sys.argv) > 1:
    KINDS = tuple(k for k in KINDS if str(k[0]) in sys.argv[1].split(","))
for kind, name in KINDS:
    for warps_per_sm in (1, 4, 8, 12, 16, 24, 32, 48, 64):
        threads = 128 if warps_per_sm >= 4 else 32 * warps_per_sm
        blocks_per_sm = max(1, warps_per_sm * 32 // threads)
        if blocks_per_sm == 0:
            continue
        iters = 300 if kind < 100 else 60
        try:
            v = ctx.op_throughput(kind, SMS * blocks_per_sm, threads, iters)
        except zk.ZkError as e:
            print(name, warps_per_sm, "failed", e)
            continue
        rows.append({"op": name, "warps_per_sm_requested": warps_per_sm, "ops_per_s": v})
        lat_us = (SMS * warps_per_sm * (8 if kind == 101 else 32 * (kind if kind < 100 else 1))) / v * 1e6   # time one warp spends per operation step
        print(f"{name:14s} warps/SM {warps_per_sm:3d}  {v:.3e} ops/s   ({v / SMS / CLOCK_HZ:.4f} per SM-clock @{CLOCK_HZ / 1e6:.0f}MHz)  step latency {lat_us:.2f} us")
json.dump(rows, open(os.path.join("gpurun_out", "microbench.json"), "w"), indent=1)
