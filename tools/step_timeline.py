"""Where the kernels of one training step run, on both streams.

One C2 step (or another bench.py config) is traced with torch.profiler (CUDA activities), once with eager launches and
once replayed as the CUDA graph SGD.step_device captures.  For every kernel, memset and copy it prints the stream
(`main` is the caller's and the training call's main chain, `side` the one libctcb200 runs the weight gradients on),
start and end in microseconds from
the step's first kernel, and the name.  Then, per BPTT sweep, the gap between the end of the main-stream kernel before
it and its start, and the side-stream time after the sweep that no main-stream kernel overlaps (the exposed part of
the recurrent weight gradients).  A graph replay runs its nodes on streams of its own, so for it only the span of the
step is reported.  The card's name and power limit are read in the same run.

    python tools/step_timeline.py [--config c2] [--out FILE]
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info  # noqa: E402
from bench import CONFIGS, make_batch  # noqa: E402


def _intervals_minus(a, b):
    """Total length of the union of intervals a not covered by the union of intervals b."""
    def union(iv):
        out = []
        for s, e in sorted(iv):
            if out and s <= out[-1][1]:
                out[-1][1] = max(out[-1][1], e)
            else:
                out.append([s, e])
        return out
    total = 0.0
    ub = union(b)
    for s, e in union(a):
        cur = s
        for bs, be in ub:
            if be <= cur or bs >= e:
                continue
            if bs > cur:
                total += bs - cur
            cur = max(cur, be)
            if cur >= e:
                break
        if cur < e:
            total += e - cur
    return total


def trace_step(torch, step):
    """The device activity of one call of step(), from a chrome trace."""
    from torch.profiler import ProfilerActivity, profile
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    acts = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    return sorted(acts, key=lambda e: e["ts"])


def analyse(acts, streams=True):
    """Summary and rows of one step's activities.  streams=False (a graph replay, whose nodes run on streams of the
    graph's own, not the ones they were captured from): the span and the count only."""
    t0 = acts[0]["ts"]
    if not streams:
        return dict(span_us=round(max(a["ts"] + a["dur"] for a in acts) - t0, 2), kernels=len(acts)), [
            dict(stream="-", start_us=round(a["ts"] - t0, 2), end_us=round(a["ts"] + a["dur"] - t0, 2),
                 name=a["name"][:90]) for a in acts]
    # `main`: the caller's stream (the step's first launch) and the one the sweeps run on (the training call's main
    # chain, forked from the caller's); `side`: every other stream
    main = {acts[0]["args"]["stream"]} | {a["args"]["stream"] for a in acts if "sweep" in a["name"]}
    rows = [dict(stream="main" if a["args"]["stream"] in main else "side", start_us=round(a["ts"] - t0, 2),
                 end_us=round(a["ts"] + a["dur"] - t0, 2), name=a["name"][:90]) for a in acts]
    mains = [(r["start_us"], r["end_us"]) for r in rows if r["stream"] == "main"]
    sweeps = [r for r in rows if "sweep" in r["name"]]
    bptt = sweeps[len(sweeps) // 2:]      # the forward sweeps come first, one per temporal layer, then the BPTT ones
    per_sweep = []
    for s in bptt:
        before = [e for (st, e) in mains if st < s["start_us"]]
        prev_end = max(before) if before else s["start_us"]
        after_side = [(r["start_us"], r["end_us"]) for r in rows if r["stream"] == "side" and r["end_us"] > s["end_us"]]
        after_side = [(max(a, s["end_us"]), b) for a, b in after_side]
        per_sweep.append(dict(start_us=s["start_us"], dur_us=round(s["end_us"] - s["start_us"], 2),
                              gap_after_main_us=round(s["start_us"] - prev_end, 2),
                              side_busy_after_us=round(_intervals_minus(after_side, []), 2),
                              side_end_after_us=round(max([b for _, b in after_side], default=s["end_us"])
                                                      - s["end_us"], 2),
                              side_exposed_after_us=round(_intervals_minus(after_side, mains), 2)))
    span = max(r["end_us"] for r in rows)
    sides = [(r["start_us"], r["end_us"]) for r in rows if r["stream"] == "side"]
    return dict(span_us=round(span, 2), kernels=len(rows), bptt=per_sweep,
                side_exposed_us=round(_intervals_minus(sides, mains), 2)), rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--config", default="c2", choices=sorted(CONFIGS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("step_timeline.py traces on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    import nnets.brnnet as rnnet
    import sgd
    c = CONFIGS[args.config]
    res = {"card": card_info(torch), "config": c["name"]}
    stream = torch.cuda.Stream()          # a stream of our own, as bench.py uses (graphs need one)
    with torch.cuda.stream(stream):
        np.random.seed(33)
        nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"],
                        maxLabels=c["L"], allowTopTemporal=c.get("top", False))
        nn.initParams()
        opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
        opt.it = 11                       # past the momentum warm-up: one step shape
        datas, labels = make_batch(c, c["B"], seed=33)
        batch = nn._batch.pack(datas, labels).upload()

        def step():
            opt.it += 1
            opt.step_device(batch, opt._momentum_now())

        for mode, graphs in (("eager", False), ("graph", True)):
            opt.useGraphs = graphs
            for _ in range(4):            # the third occurrence is captured; later ones replay
                step()
            torch.cuda.synchronize()
            summary, rows = analyse(trace_step(torch, step), streams=not graphs)
            res[mode] = summary
            print("== %s step: %d activities, %.1f us" % (mode, len(rows), summary["span_us"]))
            for r in rows:
                print("  %-4s %9.2f %9.2f %8.2f  %s" % (r["stream"], r["start_us"], r["end_us"],
                                                        r["end_us"] - r["start_us"], r["name"]))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
