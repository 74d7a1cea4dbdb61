"""What the weight average costs: training steps with emaDecay on against off, and its kernel alone.

  1. The kernel alone (ctcb_ema_update_f32) at the C4 parameter count, CUDA events over --launches launches after a
     warm-up, over --rounds rounds: 12 B per parameter (read a and w, write a), against the 0.09 ms that 12 B/param take
     at the data sheet's 3.35 TB/s.
  2. Whole optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and upload included as SGD.run does
     it) at C2 and C3, Nesterov and Adam, with emaDecay = 0 and 0.9999 alternated over --rounds rounds after a warm-up.
     The spread of the rounds is the noise to read a difference against.
The card's name, power limit and max SM clock are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/ema_time.py [--launches 200] [--steps 20] [--warmup 6] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info, make_batch, one_step, time_steps  # noqa: E402
from optim_time import HBM_BYTES_PER_S, SHAPES, param_count, time_kernel  # noqa: E402

BYTES_PER_PARAM = 12
DECAY = 0.9999


def make_opt(c, rule, decay):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"])
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, optimizer=rule, momentum=0.9, batchSize=c["B"], verbose=False,
                  emaDecay=decay)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ema_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    from _ctcb import lib, check, ptr, current_stream
    res = {"card": card_info(torch), "launches": args.launches, "steps": args.steps, "warmup": args.warmup,
           "rounds": args.rounds, "decay": DECAY, "steps_ms": {}}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    with torch.cuda.stream(stream):
        n = param_count(SHAPES["c4"])
        a, w = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
        step = torch.tensor([5000], dtype=torch.int64, device="cuda")
        nv = torch.tensor([4.0], device="cuda")
        st = current_stream()

        def ema():
            check(lib.ctcb_ema_update_f32(ptr(a), ptr(w), n, DECAY, ptr(nv), ptr(step), st))
        time_kernel(torch, ema, 10)
        ms = [time_kernel(torch, ema, args.launches) for _ in range(args.rounds)]
        best = min(ms)
        res["kernel_c4"] = dict(params=n, ms=[round(x, 5) for x in ms], bytes_per_param=BYTES_PER_PARAM,
                                bound_ms_at_3_35_TB_per_s=round(BYTES_PER_PARAM * n / HBM_BYTES_PER_S * 1e3, 5),
                                TB_per_s=round(BYTES_PER_PARAM * n / (best * 1e-3) / 1e12, 3),
                                fraction_of_3_35_TB_per_s=round(BYTES_PER_PARAM * n / (best * 1e-3) / HBM_BYTES_PER_S,
                                                                3))
        del a, w
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        for name in ("c2", "c3"):
            c = SHAPES[name]
            datas, labels = make_batch(c, c["B"], seed=33)
            out = {"shape": c}
            for rule in ("nesterov", "adam"):
                arms = {"off": make_opt(c, rule, 0.0), "on": make_opt(c, rule, DECAY)}
                for nn, opt in arms.values():
                    for _ in range(args.warmup):
                        one_step(opt, datas, labels)
                rec = {k: [] for k in arms}
                for _ in range(args.rounds):
                    for k, (nn, opt) in arms.items():
                        rec[k].append(time_steps(torch, opt, datas, labels, args.steps))
                r = {}
                for k, (nn, opt) in arms.items():
                    dev = [round(x[0], 4) for x in rec[k]]
                    r[k] = dict(ms_per_step_device=dev, ms_per_step_wall=[round(x[1], 4) for x in rec[k]],
                                spread_ms=round(max(dev) - min(dev), 4),
                                params_finite=bool(torch.isfinite(nn.params).all()))
                r["on_minus_off_ms_median"] = round(float(np.median(r["on"]["ms_per_step_device"])
                                                          - np.median(r["off"]["ms_per_step_device"])), 4)
                out[rule] = r
                del arms, nn, opt
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
            res["steps_ms"][name] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
