"""Per-launch-class ledger of the flagship step (BigGAN-Deep 256x256, the workload bench.py times).

    python profiles/conv_ledger.py --out DIR [--warmup W] [--steps K]

Builds the flagship worker through ``bench.measure(..., want_profile=True)``: W warm-up steps, K timed steps, then one
eager accounting step with CUDA events around every library call.  Prints one row per call tag (kernel class + geometry):
launches, ms, achieved TFLOP/s and GB/s (algorithmic FLOPs / bytes of the tag over its event time), the H100 SXM data-sheet
floor max(flop / 989e12, bytes / 3.35e12) and the tag's share of the timed step.  The GPU name, power limit and SM clocks
are read with a read-only ``nvidia-smi --query-gpu`` in the same run.  Everything is written to DIR/conv_ledger.json.
Load another build of the library with SGB_LIB to compare two builds.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import torch  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12      # H100 SXM data sheet: dense bf16, HBM3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,driver_version"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()
    return [dict(zip(q.split(","), (s.strip() for s in line.split(",")))) for line in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory for conv_ledger.json")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    sys.argv = ["bench.py", "--no-fid", "--no-also", "--no-cpu-baseline", "--no-e2e"]
    args = bench.parse()
    torch.cuda.set_device(0)
    device = torch.device("cuda", 0)
    from sgb200 import _lib
    _lib.check(_lib.load().sgb_device_check(), "sgb_device_check")
    info_before = gpu_info()
    res = bench.measure(args, 0, 1, device, None, a.steps, a.warmup, False, True)
    info_after = gpu_info()
    ms_step = res["ms_step"]
    by_tag = res["prof_by_tag"] or {}
    rows = []
    for tag, (ms, flop, n, nbytes) in by_tag.items():
        floor_ms = max(flop / PEAK_FLOPS, nbytes / PEAK_BYTES) * 1e3
        rows.append({"tag": tag, "class": tag.split(" ")[0], "launches": n, "ms": ms,
                     "tflops": flop / (ms * 1e-3) * 1e-12 if ms > 0 else None,
                     "gb_per_s": nbytes / (ms * 1e-3) * 1e-9 if ms > 0 else None,
                     "floor_ms": floor_ms, "share_of_step": ms / ms_step, "flop": flop, "bytes": nbytes})
    rows.sort(key=lambda r: -r["ms"])
    classes = {}
    for r in rows:
        c = classes.setdefault(r["class"], {"launches": 0, "ms": 0.0, "floor_ms": 0.0, "flop": 0.0, "bytes": 0.0})
        for k in ("launches", "ms", "floor_ms", "flop", "bytes"):
            c[k] += r[k]
    for c in classes.values():
        c["share_of_step"] = c["ms"] / ms_step
    print("step %.1f ms, %.1f img/s; accounting step (eager, events per call) %.1f ms in library calls"
          % (ms_step, res["value"], sum(r["ms"] for r in rows)))
    print("gpu: %s" % info_after)
    print("%-52s %6s %9s %8s %8s %9s %6s" % ("tag", "calls", "ms", "TFLOP/s", "GB/s", "floor ms", "share"))
    for name, c in sorted(classes.items(), key=lambda kv: -kv[1]["ms"]):
        print("%-52s %6d %9.2f %8.1f %8.1f %9.2f %5.1f%%" % ("[class] " + name, c["launches"], c["ms"],
              c["flop"] / (c["ms"] * 1e-3) * 1e-12 if c["ms"] > 0 else 0.0,
              c["bytes"] / (c["ms"] * 1e-3) * 1e-9 if c["ms"] > 0 else 0.0, c["floor_ms"], 100 * c["share_of_step"]))
    for r in rows:
        if r["class"].startswith("conv"):
            print("%-52s %6d %9.2f %8.1f %8.1f %9.2f %5.1f%%" % (r["tag"][:52], r["launches"], r["ms"], r["tflops"] or 0.0,
                  r["gb_per_s"] or 0.0, r["floor_ms"], 100 * r["share_of_step"]))
    out = {"lib": _lib.LIB_PATH, "gpu_before": info_before, "gpu_after": info_after, "clocks_during_timed_steps": res["clocks"],
           "ms_step": ms_step, "img_per_s": res["value"], "images_per_step": res["images_per_step"],
           "warmup": a.warmup, "steps": a.steps, "peaks": {"bf16_flops": PEAK_FLOPS, "hbm_bytes_per_s": PEAK_BYTES},
           "classes": classes, "tags": rows}
    with open(os.path.join(a.out, "conv_ledger.json"), "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
