"""Generates tests/golden/*.npz by running the REFERENCE ITSELF in the authoring container:
  * CTC cases through oracle/_ref = the unmodified ctc_fast/ctc-loss/ctc_fast.pyx
    and ctc_fast_blankforce.pyx (compiled by oracle/build_ref.py), fed probs.astype(float64) in Fortran
    order as brnnet.py:175 does;
  * BRNN cases through oracle/brnn_oracle.py (float64 restatement of brnnet.py; the cudamat half of
    the reference is not runnable here) with the CTC inside it again served by oracle/_ref.

Run from the repo root:  python tests/golden/gen_golden.py      (needs CTC_REFERENCE_DIR)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import recipes  # noqa: E402
from oracle import build_ref, ctc_oracle, brnn_oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    assert build_ref.build() is not None, "oracle/_ref could not be built (CTC_REFERENCE_DIR unset or Cython missing?)"
    out = {}
    for name in recipes.ALL_CTC:
        probs, seq = recipes.ctc_case(name)
        nll, grad, skip = ctc_oracle.ref_ctc_loss(np.asfortranarray(probs.astype(np.float64)), seq)
        out[name + "/nll"] = np.float64(nll)
        out[name + "/skip"] = np.bool_(skip)
        st = recipes.golden_stride(*probs.shape)
        out[name + "/grad"] = grad[:, ::st].astype(np.float32)   # K x ceil(T/st)
        out[name + "/gradnorm"] = np.float64(np.linalg.norm(grad))
        print("%-36s nll=%.9f |g|=%.9f skip=%s" % (name, nll, np.linalg.norm(grad), skip))
    np.savez_compressed(os.path.join(HERE, "ctc_cases.npz"), **out)

    # blank-forced CTC through the unmodified ctc_fast_blankforce.pyx
    out = {}
    for name in recipes.ALL_BF:
        probs, seq = recipes.bf_case(name)
        nll, grad, skip = ctc_oracle.ref_ctc_loss_blankforce(np.asfortranarray(probs.astype(np.float64)), seq)
        out[name + "/nll"] = np.float64(nll)
        out[name + "/skip"] = np.bool_(skip)
        st = recipes.golden_stride(*probs.shape)
        out[name + "/grad"] = grad[:, ::st].astype(np.float32)
        out[name + "/gradnorm"] = np.float64(np.linalg.norm(grad))
        print("%-36s nll=%.9f |g|=%.9f skip=%s" % (name, nll, np.linalg.norm(grad), skip))
    np.savez_compressed(os.path.join(HERE, "blankforce_cases.npz"), **out)

    out = {}
    # (1) the reference's own CPU BRNN self-test recipe
    cfg, data, labels = recipes.rnnetcpu()
    np.random.seed(33); np.random.randn(20, 10)       # rnnetcpu.py draws data before initParams
    nn = brnn_oracle.NNet(cfg["inputDim"], cfg["outputDim"], cfg["layerSize"], cfg["numLayers"], cfg["maxBatch"],
                          temporalLayer=cfg["temporalLayer"], dtype=np.float64)
    nn.initParams()
    cost, grad, skip = nn.costAndGrad(data.astype(np.float32), labels)
    out["rnnetcpu/cost"] = np.float64(cost)
    for i, ((w, b), (dw, db)) in enumerate(zip(nn.stack, grad)):
        out["rnnetcpu/w%d" % i] = w.astype(np.float32); out["rnnetcpu/b%d" % i] = b.astype(np.float32)
        out["rnnetcpu/dw%d" % i] = dw; out["rnnetcpu/db%d" % i] = db
    print("rnnetcpu cost %.9f" % cost)

    # (2) a ragged minibatch with the clip active and L2 on: D=13, K=11, H=64, N=3, tl=2
    lens, nlabs = [37, 50, 21, 50, 8], [9, 14, 5, 20, 3]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=7)
    np.random.seed(5)
    nn = brnn_oracle.NNet(13, 11, 64, 3, 50, temporalLayer=2, reg=1e-3, dtype=np.float64)
    nn.initParams()
    for w, b in nn.stack[:-2]:
        b += 0.05
    # push the recurrence into the 20.0 clip (brnnet.py:32,146-152) through a positive drive on the
    # temporal layer rather than a super-critical recurrent matrix (which would make float32 vs float64
    # trajectories diverge chaotically and the comparison meaningless)
    nn.stack[1][1] += 4.0
    nn.stack[-2][0] *= 1.2
    nn.stack[-1][0] *= 1.2
    hA = nn.forward(datas[1])
    out["ragged/clip_hits"] = np.int64(np.sum(hA[1] >= 20.0) + np.sum(hA[2] >= 20.0))
    costs, grad, skips = nn.costAndGradBatch(datas, labelss)
    out["ragged/costs"] = costs; out["ragged/skips"] = skips; out["ragged/regcost"] = np.float64(nn.regcost)
    for i, ((w, b), (dw, db)) in enumerate(zip(nn.stack, grad)):
        out["ragged/w%d" % i] = w.astype(np.float32); out["ragged/b%d" % i] = b.astype(np.float32)
        out["ragged/dw%d" % i] = dw; out["ragged/db%d" % i] = db
    print("ragged costs", costs, "clip hits", out["ragged/clip_hits"], "regcost", nn.regcost)
    np.savez_compressed(os.path.join(HERE, "brnn_cases.npz"), **out)

    # (3) the uni-directional net (nnets/rnnet.py) and the feed-forward net (nnets/nnet.py) on a ragged minibatch
    out = {}
    datas, labelss = recipes.rnn_variant_batch()
    for tag, _ in recipes.RNN_VARIANTS:
        nn = recipes.rnn_variant_net(brnn_oracle.NNet, tag, dtype=np.float64)
        recipes.rnn_variant_perturb(nn.stack, tag)
        if tag == "uni":
            out["uni/clip_hits"] = np.int64(np.sum(nn.forward(datas[1])[1] >= 20.0))
        costs, grad, skips = nn.costAndGradBatch(datas, labelss)
        out[tag + "/costs"] = costs; out[tag + "/skips"] = skips
        for i, ((w, b), (dw, db)) in enumerate(zip(nn.stack, grad)):
            out[tag + "/w%d" % i] = w.astype(np.float32); out[tag + "/b%d" % i] = b.astype(np.float32)
            out[tag + "/dw%d" % i] = dw; out[tag + "/db%d" % i] = db
        print(tag, "costs", costs, "clip hits", out.get("uni/clip_hits"))
    np.savez_compressed(os.path.join(HERE, "rnn_cases.npz"), **out)


if __name__ == "__main__":
    main()
