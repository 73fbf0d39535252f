#!/usr/bin/env python
"""Per-kernel split of one captured E+F evaluation (CUDA-graph replay), from a torch.profiler trace.

    python tools/profile_kernels.py --config cfg2 --steps 20 --out DIR

The kernels are chained by programmatic dependent launch: each one starts while its predecessor is still running and
waits in griddepcontrol.wait, so a kernel's own start-to-end span counts its predecessor's tail.  The time charged to a
kernel here is therefore the time the stream's last completion advanced when it ended,
``end_k - max(end_{k-1}, start_k)``; these sum to the replay's busy time.  Launches are grouped by kernel name and grid,
which for ``k_dense_tc`` identifies the layer shape (grid = [ceil(M/128), ceil(N/TN)]).  Run on its own: tracing slows
the host, so end-to-end step times come from bench.py, not from here.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec  # noqa: E402


def short_name(name: str) -> str:
    """`void (anonymous namespace)::k_dense_tc<128, 0, 1>(...)` -> `k_dense_tc<128, 0, 1>`"""
    name = re.sub(r"^void\s+", "", name)
    name = name.replace("(anonymous namespace)::", "")
    depth, out = 0, []
    for ch in name:                       # drop the parameter list, keep template arguments
        if ch == "(" and depth == 0:
            break
        depth += ch == "<"
        depth -= ch == ">"
        out.append(ch)
    return "".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", required=True, help="directory for the trace and the JSON summary")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_kernels.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    spec, data = S.make_config(args.config, seed=0) if args.config in ("cfg2", "cfg3") else S.make_config(args.config)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    g = GraphedPotential(model)
    g(batch_to_device(data, dev))
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            g.replay()
            torch.cuda.synchronize()       # separates the replays in the trace
    trace = os.path.join(args.out, f"trace_{args.config}.pt.trace.json")
    prof.export_chrome_trace(trace)
    ev = [e for e in json.load(open(trace))["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: e["ts"])
    if not ev:
        raise SystemExit("no kernel activity in the trace")

    # split into replays at the host synchronisations (gaps far longer than any in-graph gap)
    steps, cur = [], [ev[0]]
    for e in ev[1:]:
        if e["ts"] - max(x["ts"] + x["dur"] for x in cur) > 50.0:
            steps.append(cur)
            cur = []
        cur.append(e)
    steps.append(cur)
    steps = [s for s in steps if len(s) == len(steps[-1])]   # complete replays only

    per = defaultdict(list)   # (name, grid) -> incremental us, all launches of all replays
    step_us = []
    for s in steps:
        last_end = s[0]["ts"]
        for e in s:
            end = e["ts"] + e["dur"]
            inc = max(0.0, end - max(last_end, e["ts"]))
            last_end = max(last_end, end)
            grid = tuple(e.get("args", {}).get("grid", ()))
            per[(short_name(e["name"]), grid)].append(inc)
        step_us.append(last_end - s[0]["ts"])
    n = len(steps)
    rows = []
    for (name, grid), v in per.items():
        rows.append({"kernel": name, "grid": list(grid), "launches_per_step": len(v) / n, "us_per_step": sum(v) / n,
                     "us_per_launch": sum(v) / len(v)})
    rows.sort(key=lambda r: -r["us_per_step"])
    busy = sum(step_us) / n
    dense = [r for r in rows if r["kernel"].startswith("k_dense_tc")]
    dense_us = sum(r["us_per_step"] for r in dense)
    props = torch.cuda.get_device_properties(0)
    summary = {"config": args.config, "replays": n, "kernels_per_step": len(steps[-1]), "busy_us_per_step": busy,
               "dense_tc_us_per_step": dense_us, "dense_tc_launches_per_step": sum(r["launches_per_step"] for r in dense),
               "dense_tc_share": dense_us / busy, "gpu": props.name, "rows": rows}
    try:
        import subprocess

        summary["nvidia_smi"] = subprocess.run(
            ["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        pass
    json.dump(summary, open(os.path.join(args.out, f"kernels_{args.config}.json"), "w"), indent=1)
    print(f"{props.name}  {summary.get('nvidia_smi', '')}")
    print(f"{args.config}: {n} replays, {len(steps[-1])} kernels, busy {busy:.1f} us/step; "
          f"k_dense_tc {dense_us:.1f} us/step ({100 * dense_us / busy:.1f} %) in "
          f"{summary['dense_tc_launches_per_step']:.0f} launches")
    for r in rows[:40]:
        print(f"{r['us_per_step']:9.1f} us  {r['launches_per_step']:4.1f} x {r['us_per_launch']:7.2f} us  "
              f"{r['kernel']}  grid={r['grid']}")


if __name__ == "__main__":
    main()
