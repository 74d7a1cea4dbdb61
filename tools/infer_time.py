"""Inference throughput of NNet.forwardBatch (the batched likelihood writer's forward pass) against utterances per call.

For C2 (H=512, N=2, T=200), C3 (H=1024, N=3, T=800) and a C4-width net (H=2048, N=5, T=1500), random weights, the
same set of ragged utterances (lengths uniform in [T/2, T]; 2048, 512 and 256 of them, so that the batched arms
run for a fair fraction of a second) goes through forwardBatch at maxUtts = 1 (the reference's
one-utterance loop), 32 and 128.  A timing covers everything the writer waits for: sorting, host packing, H2D, the
forward calls, D2H of the probabilities and the per-micro-batch synchronisation (host clock around the call, which
ends synchronised).  Warm-up pass first; the arms alternate over --rounds rounds and the best round counts.  The
card's name and power limit are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/infer_time.py [--rounds 2] [--configs C2,C3,C4_width] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info  # noqa: E402

CONFIGS = {
    "C2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, utts=2048),
    "C3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, utts=512),
    "C4_width": dict(D=41, K=35, H=2048, N=5, tl=3, T=1500, utts=256),
}
MAX_UTTS = (1, 32, 128)


def make_net(c, maxUtts):
    import nnets.brnnet as rnnet
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], train=False, temporalLayer=c["tl"], maxUtts=maxUtts)
    nn.initParams()
    return nn


def workspace_bytes(c, maxB):
    from _ctcb import lib, BrnnConfig
    cfg = BrnnConfig(c["D"], c["K"], c["H"], c["N"], c["tl"], c["T"], maxB, 0, 0.0, 20.0, 0)
    return {"forward": int(lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None)),
            "training": int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)))}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("infer_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "rounds": args.rounds}
    for name in args.configs.split(","):
        c = CONFIGS[name]
        rng = np.random.RandomState(7)
        lens = [int(x) for x in rng.randint(c["T"] // 2, c["T"] + 1, size=c["utts"])]
        datas = [rng.randn(c["D"], T).astype(np.float32) for T in lens]
        nets = {m: make_net(c, m) for m in MAX_UTTS}
        outs = {m: nets[m].forwardBatch(datas) for m in MAX_UTTS}         # warm-up (and the outputs compared below)
        times = {m: [] for m in MAX_UTTS}
        for _ in range(args.rounds):
            for m in MAX_UTTS:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                nets[m].forwardBatch(datas)
                times[m].append(time.perf_counter() - t0)
        best = {m: min(ts) for m, ts in times.items()}
        rec = {"utterances": len(lens), "frames": int(sum(lens)),
               "workspace_bytes": {m: workspace_bytes(c, m) for m in MAX_UTTS}}
        for m in MAX_UTTS:
            rec["maxUtts_%d" % m] = dict(
                seconds=round(best[m], 4), seconds_per_round=[round(t, 4) for t in times[m]],
                utts_per_s=round(len(lens) / best[m], 1),
                speedup_vs_maxUtts_1=round(best[1] / best[m], 2),
                max_abs_prob_diff_vs_maxUtts_1=float(max(np.abs(a - b).max() for a, b in zip(outs[m], outs[1]))))
        res[name] = rec
        del nets, outs
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
