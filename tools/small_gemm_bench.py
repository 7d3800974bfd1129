"""Per-call cost of the small-map implicit-GEMM convolutions of bench.py's engine.

    python tools/small_gemm_bench.py [--lib path/to/libdvmvs_sm90.so] [--json out.json]

Builds bench.py's default engine (tools/engine_record.engine_calls), keeps every dvmvs_conv2d_tc call whose output map has at
most 32x32 pixels per image, and replays each one alone at its shape and with its outputs, captured in a CUDA graph
(tools/tc_bench.graph_timeit).  Per call it reports: us per call (GEMM + finishing pass), the packed fp16 weight bytes the call
streams (all operand planes) and the GB/s of weights that makes, the GEMM kernel's grid (CTAs, from a torch.profiler trace of
one call) and CTA x us (grid x the GEMM kernel's profiled time), and whether the engine runs it on its recurrent stage.
--lib loads another build of the library (an A/B comparison of two builds in one process is not possible: one per run)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
import torch

from dvmvs import _native as N
from dvmvs import _ops as ops

MAX_PIXELS = 32 * 32


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name(0) + ", power limit not read"
    return q


def gemm_kernels(fn):
    """[(kernel name, CTAs, us)] of the kernels one call of fn launches, from a torch.profiler trace"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            events = json.load(fh)["traceEvents"]
    out = []
    for e in sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"]):
        g = e.get("args", {}).get("grid", [1, 1, 1])
        out.append((e["name"], int(g[0]) * int(g[1]) * int(g[2]), float(e["dur"])))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.lib:
        N.LIB_PATH = os.path.abspath(args.lib)
    from tools.engine_record import engine_calls, layer_names
    from tools.tc_bench import graph_timeit
    hw = card()
    mods, calls = engine_calls(("conv2d_tc",))
    names = layer_names(mods)
    rows = []
    with torch.no_grad():
        for key, (a, kw, lay, on_rec) in calls.items():
            planes, ptc = a[0], a[1]
            B, Hin, Win = planes[0].shape[1], planes[0].shape[2], planes[0].shape[3]
            pad = (ptc.ksize - 1) // 2
            Ho, Wo = (Hin + 2 * pad - ptc.ksize) // ptc.stride + 1, (Win + 2 * pad - ptc.ksize) // ptc.stride + 1
            if Ho * Wo > MAX_PIXELS:
                continue
            fn = lambda: ops.conv2d_tc(*a, **kw)      # noqa: E731
            t = graph_timeit(fn)
            kern = gemm_kernels(fn)
            main_k = next((k for k in kern if k[0].startswith(("void dvmvs::conv_tc_kernel", "void dvmvs::conv_ws_kernel"))),
                          kern[0] if kern else ("?", 0, 0.0))
            terms = kw.get("terms", 3)
            w_bytes = ptc.cout * ptc.ktot * 2 * (2 if terms == 3 else 1)        # the rows a call streams (padding rows excluded)
            rows.append({"layer": names.get(id(lay), "?"), "recurrent": on_rec, "B": B, "Hout": Ho, "Wout": Wo, "sources": [int(p.shape[4]) for p in planes],
                         "cout": ptc.cout, "k": ptc.ksize, "stride": ptc.stride, "terms": terms, "deferred_finish": bool(kw.get("defer_finish")),
                         "us": t, "weight_mb": w_bytes / 1e6, "weight_gbs": w_bytes / (t * 1e-6) / 1e9,
                         "kernel": main_k[0].split("(")[0].replace("void dvmvs::", ""), "ctas": main_k[1], "kernel_us": main_k[2],
                         "cta_us": main_k[1] * main_k[2], "kernels": [k[0].split("(")[0].replace("void dvmvs::", "") for k in kern]})
    rows.sort(key=lambda r: (not r["recurrent"], -r["us"]))
    print("card:", hw)
    print("library:", N.LIB_PATH)
    for r in rows:
        print("%-26s %s B=%-2d %2dx%-2d s%d %-14s->%-4d k%d %8.2f us %6.2f MB %7.0f GB/s  %-22s %4d CTAs x %6.2f us = %7.0f CTA.us" % (
            r["layer"], "rec" if r["recurrent"] else "   ", r["B"], r["Hout"], r["Wout"], r["stride"], "+".join(map(str, r["sources"])),
            r["cout"], r["k"], r["us"], r["weight_mb"], r["weight_gbs"], r["kernel"], r["ctas"], r["kernel_us"], r["cta_us"]))
    rec = [r for r in rows if r["recurrent"]]
    summary = {"card": hw, "library": N.LIB_PATH, "timing": "graph_timeit",
               "recurrent_us": sum(r["us"] for r in rec), "recurrent_cta_us": sum(r["cta_us"] for r in rec),
               "all_us": sum(r["us"] for r in rows), "all_cta_us": sum(r["cta_us"] for r in rows), "calls": rows}
    print("recurrent stage: %.1f us, %.0f CTA.us;  all small-map calls: %.1f us, %.0f CTA.us" % (
        summary["recurrent_us"], summary["recurrent_cta_us"], summary["all_us"], summary["all_cta_us"]))
    print(json.dumps({k: v for k, v in summary.items() if k != "calls"}))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(summary, fh, indent=1)


if __name__ == "__main__":
    main()
