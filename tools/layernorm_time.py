"""What layer normalisation costs: whole steps with it off and on, and its two kernels alone.

Two shapes: C2 (H=512, numLayers=2, temporalLayer=1, B=32, T=200: one normalised layer of 6400 x 512) and C3 (H=1024,
numLayers=3, temporalLayer=2, B=128, T=800: two of 102400 x 1024), each built with layerNorm off and on.  Each arm is
timed over whole optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and upload included as
SGD.run does it), the arms alternated over two rounds after a warm-up.  Then ctcb_layernorm_forward_f32 (with the row
statistics) and ctcb_layernorm_backward_f32 at each shape's normalised-layer size, alone, over --launches launches
between CUDA events: algorithmic bytes are the forward's z read and X written, the backward's g and z read and dz
written (4 B per element each), plus the row statistics (8 B per row, written by the forward and read by the backward)
and, for the backward, its partial sums written and read once; bytes/s is those bytes over the kernel time.  The card's
name, power limit and clock are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/layernorm_time.py [--steps 5] [--warmup 4] [--launches 200] [--shapes c2,c3] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info, make_batch, one_step, time_steps  # noqa: E402

SHAPES = {
    "c2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32),
    "c3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100, B=128),
}


def make_opt(c, layerNorm):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                    layerNorm=layerNorm)
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def time_kernels(torch, R, H, launches):
    """Each kernel alone at R x H, best of three windows of `launches` launches."""
    from _ctcb import lib, check
    g = torch.Generator(device="cuda").manual_seed(1)
    z = torch.randn(R * H, device="cuda", generator=g)
    d0 = torch.randn(R * H, device="cuda", generator=g)
    y = torch.empty_like(z)
    d = d0.clone()
    mu = torch.empty(R, device="cuda")
    rstd = torch.empty_like(mu)
    gamma = torch.ones(H, device="cuda")
    beta = torch.zeros(H, device="cuda")
    dgamma, dbeta = torch.empty_like(gamma), torch.empty_like(beta)
    ws_bytes = int(lib.ctcb_layernorm_workspace_bytes(R, H))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def fwd():
        check(lib.ctcb_layernorm_forward_f32(z.data_ptr(), y.data_ptr(), mu.data_ptr(), rstd.data_ptr(),
                                             gamma.data_ptr(), beta.data_ptr(), R, H, st))

    def bwd():     # in place on d: its values drift over the launches, its traffic does not
        check(lib.ctcb_layernorm_backward_f32(d.data_ptr(), z.data_ptr(), mu.data_ptr(), rstd.data_ptr(),
                                              gamma.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), R, H, 0,
                                              ws.data_ptr(), ws_bytes, st))

    parts = -(-R // max(8, -(-R // 1024)))
    nbytes = {"forward": 8 * R * H + 8 * R, "backward": 12 * R * H + 8 * R + 2 * (2 * parts * H * 4)}
    out = {}
    for name, fn in (("forward", fwd), ("backward", bwd)):
        for _ in range(10):
            fn()
        best = None
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                fn()
            e1.record()
            e1.synchronize()
            ms = e0.elapsed_time(e1) / launches
            best = ms if best is None else min(best, ms)
        out[name] = dict(us=round(best * 1e3, 2), bytes=nbytes[name], TBps=round(nbytes[name] / (best * 1e-3) / 1e12, 3))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--shapes", default="c2,c3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("layernorm_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "steps": args.steps, "warmup": args.warmup, "launches": args.launches,
           "shapes": {}}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    for name in args.shapes.split(","):
        c = SHAPES[name]
        datas, labels = make_batch(c, c["B"], seed=33)
        out = {}
        with torch.cuda.stream(stream):
            arms = {ln: make_opt(c, ln) for ln in (False, True)}
            for ln, (nn, opt) in arms.items():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
            rec = {ln: [] for ln in arms}
            for _ in range(2):                   # alternate the arms: two rounds each
                for ln, (nn, opt) in arms.items():
                    rec[ln].append(time_steps(torch, opt, datas, labels, args.steps))
            from _ctcb import lib
            for ln, (nn, opt) in arms.items():
                out["on" if ln else "off"] = dict(
                    ms_per_step_device=[round(r[0], 3) for r in rec[ln]],
                    ms_per_step_wall=[round(r[1], 3) for r in rec[ln]],
                    params=nn.nparams,
                    workspace_bytes=int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(nn._cfg))),
                    params_finite=bool(torch.isfinite(nn.params).all()),
                    normalised_layers=nn.normedLayers())
            off, on = min(r[0] for r in rec[False]), min(r[0] for r in rec[True])
            out["on_minus_off_ms"] = round(on - off, 3)
            out["on_over_off_step"] = round(on / off, 4)
            del arms
            torch.cuda.empty_cache()
            out["kernels"] = time_kernels(torch, c["T"] * c["B"], c["H"], args.launches)
        res["shapes"][name] = dict(shape=c, arms=out)
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
