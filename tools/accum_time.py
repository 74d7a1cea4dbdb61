"""What gradient accumulation costs, and a step that needs it.

  1. One C3-shaped step (H=1024, N=3, B=128, T=800) timed as ONE call of 128 utterances and as FOUR accumulated
     micro-batches of 32 (sgd.SGD.step_device / step_device_parts, each step packed and uploaded on the host as
     SGD.run does), alternating the two arms over two rounds; CUDA events on the launching stream, warm-up first.
  2. C4 (H=2048, N=5, B=256, T=1500) on ONE GPU with buffers sized for the reference's default maxUttLen = 5000:
     one call would need the workspace printed below, so it runs as 8 micro-batches of 32.

The card's name and power limit are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/accum_time.py [--steps 5] [--warmup 6] [--no-c4] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200")]

import numpy as np  # noqa: E402

C3 = dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100)
C4 = dict(D=41, K=35, H=2048, N=5, tl=3, T=1500, L=150)


def card_info(torch):
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [x.strip() for x in out.split(",")[:2]]
    except Exception as e:      # the number is then reported without it, and says so
        info["power_limit"] = "not read (%s)" % type(e).__name__
    return info


def make_batch(c, n, seed):
    rng = np.random.RandomState(seed)
    datas = [rng.randn(c["D"], c["T"]).astype(np.float32) for _ in range(n)]
    labels = [(1 + np.floor(rng.rand(c["L"]) * (c["K"] - 1))).astype(np.int32) for _ in range(n)]
    return datas, labels


def make_opt(c, maxT, maxUtts, batchSize):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], maxT, temporalLayer=c["tl"], maxUtts=maxUtts, maxLabels=c["L"])
    nn.initParams()
    opt = sgd.SGD(nn, maxT, alpha=1e-5, momentum=0.9, batchSize=batchSize, verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def workspace_bytes(c, maxT, maxB):
    from _ctcb import lib, BrnnConfig
    cfg = BrnnConfig(c["D"], c["K"], c["H"], c["N"], c["tl"], maxT, maxB, c["L"], 0.0, 20.0, 0)
    return int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)))


def one_step(opt, datas, labels):
    """One optimisation step as SGD.run issues it: host packing and upload included, no synchronisation."""
    import parallel
    nn = opt.model
    opt.it += 1
    if len(datas) > nn.maxUtts:
        opt.step_device_parts(parallel.micro_batches(list(zip(datas, labels)), nn.maxUtts), 0.9)
    else:
        opt.step_device(nn.swap_batches().pack(datas, labels).upload(), 0.9)


def time_steps(torch, opt, datas, labels, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    for _ in range(steps):
        one_step(opt, datas, labels)
    e1.record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return e0.elapsed_time(e1) / steps, 1e3 * wall / steps


def phase_profile(torch, opt, datas, labels, nprof=2):
    """Per-phase device time of one step (CUDA events inside libctcb200 around every phase), summed over the
    micro-batches of the step; eager launches, since the events need them."""
    from _ctcb import lib, check
    graphs, opt.useGraphs = opt.useGraphs, False
    torch.cuda.synchronize()
    lib.ctcb_profile_enable(1)
    for _ in range(nprof):
        one_step(opt, datas, labels)
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 16)
    check(lib.ctcb_profile_report(buf, len(buf)))
    lib.ctcb_profile_enable(0)
    opt.useGraphs = graphs
    return {k: round(v["total_ms"] / nprof, 2) for k, v in json.loads(buf.value.decode()).items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--c4-steps", type=int, default=3)
    ap.add_argument("--no-c4", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("accum_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch)}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    with torch.cuda.stream(stream):
        # ---- 1. C3 step: 1 x 128 against 4 x 32
        datas, labels = make_batch(C3, 128, seed=33)
        arms = {"1x128": make_opt(C3, C3["T"], 128, 128), "4x32": make_opt(C3, C3["T"], 32, 128)}
        for name, (nn, opt) in arms.items():
            for _ in range(args.warmup):
                one_step(opt, datas, labels)
        rec = {name: [] for name in arms}
        for _ in range(2):                   # alternate the arms: two rounds each
            for name, (nn, opt) in arms.items():
                rec[name].append(time_steps(torch, opt, datas, labels, args.steps))
        p1, p4 = (arms[k][0].params.cpu().numpy().astype(np.float64) for k in ("1x128", "4x32"))
        c3 = {name: dict(ms_per_step_device=[round(r[0], 3) for r in rs], ms_per_step_wall=[round(r[1], 3) for r in rs])
              for name, rs in rec.items()}
        for name, (nn, opt) in arms.items():     # where the time goes: per-phase events, an untimed eager pass
            c3[name]["phases_ms"] = phase_profile(torch, opt, datas, labels)
        best1 = min(r[0] for r in rec["1x128"])
        best4 = min(r[0] for r in rec["4x32"])
        c3["overhead_of_accumulating"] = round(best4 / best1 - 1.0, 4)
        c3["params_rel_diff_after_all_steps"] = float(np.linalg.norm(p4 - p1) / np.linalg.norm(p1))
        c3.update(steps=args.steps, warmup=args.warmup, workspace_bytes={
            "1x128": workspace_bytes(C3, C3["T"], 128), "4x32": workspace_bytes(C3, C3["T"], 32)})
        res["c3_B128_T800"] = c3
        del arms, nn, opt
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

        # ---- 2. C4, batch 256 on one GPU, buffers for maxUttLen 5000, as 8 x 32
        if not args.no_c4:
            maxT = 5000
            c4 = {"workspace_bytes_1x256": workspace_bytes(C4, maxT, 256),
                  "workspace_bytes_8x32": workspace_bytes(C4, maxT, 32),
                  "device_memory_bytes": torch.cuda.get_device_properties(0).total_memory}
            datas, labels = make_batch(C4, 256, seed=44)
            nn, opt = make_opt(C4, maxT, 32, 256)
            for _ in range(2):
                one_step(opt, datas, labels)
            ms, wall = time_steps(torch, opt, datas, labels, args.c4_steps)
            rec = nn.record.cpu().numpy()
            c4.update(completed=bool(np.isfinite(nn.params.cpu().numpy()).all() and rec[3] == 0),
                      n_valid=float(rec[0]), n_skipped=float(rec[2]), ms_per_step_device=round(ms, 1),
                      ms_per_step_wall=round(wall, 1), steps=args.c4_steps, warmup=2,
                      peak_allocated_bytes=torch.cuda.max_memory_allocated())
            res["c4_B256_T1500_maxUttLen5000_8x32"] = c4
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
