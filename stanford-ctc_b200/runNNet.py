"""runNNet -- training / likelihood-dump driver for the H100 backend.

Call surface kept from the reference driver (ctc_fast/runNNet.py:23-237): `run(args)` and
`test(opts)`, every command-line flag of runNNet.py:27-69 with its default, the run-directory protocol
(cfg.json, params.pk = SGD pickle followed by the stack pickle, params.pk.epochNN, epoch, num_files,
last_cost, sentinel, train.log), resume through --cfg_file with the step size re-annealed
(runNNet.py:143-166), the fixed seeds 33 (:113-115) and CUDA_DEVICE device selection (:117-120).
The implementation is organised differently: a declarative flag table, one RunDir helper that owns the
side files, and separate train/evaluate phases.  Site paths of run_cfg.py / decoder_config.py became
flags (--runDir, --outDir); new flags: --numTemporal, --cell, --peephole, --layerNorm, --subsample, --subsampleLayer, --batchSize, --maxUtts, --maxLabels,
--dropout, --freqMasks, --freqMaskWidth, --timeMasks, --timeMaskWidth, --timeMaskRatio, --featDim, --weightNoise,
--zoneoutCell, --zoneoutHidden, --interLayer, --interWeight, --selfCondition, --tf32,
--optimizer,
--beta1, --beta2, --epsilon, --emaDecay, --lastWeights, --quiet.  With --emaDecay, params.pk holds a third pickle,
the weight average in the stack's format.  Under torchrun the same
script trains data-parallel (one process per GPU, one NCCL all-reduce per step).
"""
import argparse
import logging
import os
import pickle
import random
import time

import numpy as np

import dataLoader as dl
import nnets.brnnet as rnnet
import parallel
import sgd
from run_utils import CfgStruct, TimeString, dump_config, get_git_revision, get_hostname, load_config, touch_file
from writeLikelihoods import writeLogLikes

MAX_UTT_LEN = 5000   # default of the reference (decoder/decoder_config.py:28, DATASET == 'swbd')

# (flag, type, default, help); None type = boolean switch.  Names and defaults: runNNet.py:27-69.
FLAGS = [
    ("cfg_file", str, None, "cfg.json of an earlier run: resume training / select the model for --test"),
    ("test", None, False, "forward-only pass that writes log-likelihood arks"),
    ("layerSize", int, 1824, None), ("numLayers", int, 5, None), ("temporalLayer", int, 3, None),
    ("momentum", float, 0.95, None), ("epochs", int, 20, None), ("step", float, 1e-5, None),
    ("anneal", float, 1.3, "learning rate := learning rate / anneal after each epoch"),
    ("reg", float, 0.0, "lambda of the L2 penalty on the weight matrices"),
    ("dataDir", str, "./data/", None), ("alisDir", str, None, None),
    ("startFile", int, 1, "first file in --test mode"), ("numFiles", int, 384, None),
    ("inputDim", int, 41 * 15, None), ("rawDim", int, 41 * 15, None), ("outputDim", int, 35, None),
    ("maxUttLen", int, MAX_UTT_LEN, None),
    ("save_every", int, 10, "checkpoint every this many data files"),
    ("run_desc", str, "", "free-text description stored in cfg.json"),
    # additions
    ("numTemporal", int, 1, "stacked temporal layers: layers temporalLayer .. temporalLayer+numTemporal-1 are all "
                            "recurrent (1 = the reference's single temporal layer)"),
    ("cell", str, "relu", "recurrence of the temporal layers: relu (the reference's clipped ReLU) or lstm; a cfg.json "
                          "written without it is relu"),
    ("peephole", None, False, "peephole connections of the LSTM cell (needs --cell lstm; the cell of Graves' TIMIT and "
                              "EESEN models); a cfg.json written without it has none"),
    ("layerNorm", None, False, "layer normalisation of the ReLU hidden layers (gamma * layer_norm(z) + beta, then "
                               "ReLU); a cfg.json written without it has none"),
    ("subsample", int, 1, "k >= 2: map --subsampleLayer reads k consecutive frames of the layer below it, and it and "
                          "every layer above run at 1/k of the frame rate (the arks of --test too); 1 = off, and a "
                          "cfg.json written without it"),
    ("subsampleLayer", int, 1, "the affine map (1..numLayers+1) that reads the stacked frames when --subsample >= 2"),
    ("batchSize", int, 1, "utterances per optimisation step (1 = the reference schedule)"),
    ("maxUtts", int, 0, "utterances per micro-batch per GPU: a larger shard accumulates its gradient over several "
                        "micro-batches (0 = the whole shard, batchSize / number of GPUs rounded up); with --test, "
                        "utterances per forward call per GPU (0 = one, the reference's loop)"),
    ("maxLabels", int, 511, "longest label sequence the buffers are sized for"),
    ("dropout", float, 0.0, "inverted dropout probability on the ReLU hidden layers while training (0 = off; "
                            "--test never drops)"),
    ("freqMasks", int, 0, "SpecAugment while training: frequency masks per utterance and step, each a band of at most "
                          "--freqMaskWidth filter-bank bins of every frame slot (0 = off; --test never masks; a cfg.json "
                          "written without it has none)"),
    ("freqMaskWidth", int, 0, "widest frequency mask, in bins (at most --featDim)"),
    ("timeMasks", int, 0, "SpecAugment while training: time masks per utterance and step, each a span of raw frames"),
    ("timeMaskWidth", int, 0, "widest time mask, in frames"),
    ("timeMaskRatio", float, 1.0, "a time mask covers at most this fraction of the utterance's frames"),
    ("featDim", int, None, "filter-bank bins per frame slot of the spliced input (e.g. 41 for --inputDim 41*15); "
                           "default --inputDim, features without splicing"),
    ("weightNoise", float, 0.0, "standard deviation of the Gaussian noise added to the weight matrices while training, "
                                "one draw per step (0 = off; --test never adds noise; a cfg.json written without it "
                                "has none)"),
    ("zoneoutCell", float, 0.0, "zoneout probability of the LSTM cell state c while training (needs --cell lstm; "
                                "0 = off; --test runs the expectation cell with the trained value; a cfg.json "
                                "written without it has none)"),
    ("zoneoutHidden", float, 0.0, "zoneout probability of the LSTM output h, as --zoneoutCell"),
    ("interLayer", int, 0, "intermediate CTC loss while training: hidden layer m (1..numLayers-1) through the output "
                           "map, scored against the same labels (0 = off; --test ignores it without "
                           "--selfCondition; a cfg.json written without it has none)"),
    ("interWeight", float, 0.0, "lambda of the intermediate CTC loss: the objective is main + lambda * intermediate "
                                "(Lee & Watanabe's weight w is lambda = w / (1 - w) at (1 - w) times the step size)"),
    ("selfCondition", None, False, "self-conditioned CTC (needs --interLayer): the intermediate posteriors, projected "
                                   "back to the layer's width, are added to layer m's output, in training and in --test "
                                   "alike; a cfg.json written without it has none"),
    ("tf32", None, False, "TF32 mode: the tensor-core contractions and sweeps read their operands rounded to TF32 and "
                          "run one MMA per product instead of three (PyTorch's allow_tf32), in training and in --test "
                          "alike; checkpoints are the same in both modes; a cfg.json written without it is off"),
    ("optimizer", str, "nesterov", "update rule: nesterov (the reference's, with --momentum), adagrad or adam; --step "
                                   "is the step size of each and --anneal applies to it"),
    ("beta1", float, 0.9, "adam: decay of the first-moment estimate"),
    ("beta2", float, 0.999, "adam: decay of the second-moment estimate"),
    ("epsilon", float, 1e-8, "adam: added to the square root of the second moment"),
    ("emaDecay", float, 0.0, "decay d in [0, 1) of an exponential moving average of the weights, updated every step "
                             "(the mean of the iterates until step 1/(1-d), then the EMA); checkpoints carry it as a "
                             "third pickle of params.pk and --test writes the arks from it (0 = off; a cfg.json written "
                             "without it has none)"),
    ("lastWeights", None, False, "--test of a run trained with --emaDecay: write the arks from the last weights, not "
                                 "from the average (taken from the command line, not from cfg.json)"),
    ("runDir", str, "./runs", "parent of the time-stamped run directory"),
    ("outDir", str, None, "--test: directory for the likelihood arks"),
    ("quiet", None, False, "no console logging / per-iteration prints"),
]


def _parse(argv):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    for name, typ, default, hlp in FLAGS:
        if typ is None:
            ap.add_argument("--" + name, dest=name, action="store_true", default=default, help=hlp)
        else:
            ap.add_argument("--" + name, dest=name, type=typ, default=default, help=hlp)
    return ap.parse_args(argv)


def run_config(cli):
    """The run's configuration: the command line of a new run, or the cfg.json of the run being resumed (its flags
    win, so a resumed run keeps e.g. its batchSize and maxUtts), with the defaults of keys an older run did not
    record."""
    cfg = load_config(cli.cfg_file) if cli.cfg_file is not None else dict(vars(cli))
    for name, _, default, _ in FLAGS:                 # configs written by older runs lack the new keys
        cfg.setdefault(name, default)
    return cfg


def trained_config(cfg_file):
    """The stored configuration of a trained model, with the defaults of keys an older run did not record (a model
    from before --numTemporal has one temporal layer)."""
    cfg = load_config(cfg_file)
    for name, _, default, _ in FLAGS:
        cfg.setdefault(name, default)
    return CfgStruct(**cfg)


def utterance_capacity(opts, world):
    """Utterances per micro-batch this process's net is built for (--maxUtts, default the whole shard)."""
    return parallel.micro_batch_capacity(opts.maxUtts, opts.batchSize, world)


def _select_device():
    """One process per GPU: LOCAL_RANK under torchrun, else the reference's CUDA_DEVICE variable."""
    import torch
    import torch.distributed as dist
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and "RANK" in os.environ:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        if not dist.is_initialized():
            dist.init_process_group(backend="nccl")
        return dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(int(os.environ.get("CUDA_DEVICE", 0)))
    return 0, 1


class RunDir(object):
    """The files a run leaves behind, under the names the reference's tools (browse_runs.py, reboot_runs.py,
    plot_results.py) look for."""

    def __init__(self, path):
        self.path = path

    def file(self, name):
        return os.path.join(self.path, name)

    def read_int(self, name, default):
        f = self.file(name)
        return int(open(f).read().strip()) if os.path.exists(f) else default

    def write(self, name, value):
        with open(self.file(name), "w") as fid:
            fid.write(str(value))

    def checkpoint(self, optimizer, net, suffix=""):
        # two pickles back to back, the SGD state and the stack; with a weight average, the average as a third
        with open(self.file("params.pk") + suffix, "wb") as fid:
            optimizer.toFile(fid)
            net.toFile(fid)
            if optimizer.average is not None:
                optimizer.averageToFile(fid)


def _attach_logging(run, rank, quiet):
    root = logging.getLogger()
    root.setLevel(logging.DEBUG)
    for old in [h for h in root.handlers if getattr(h, "_ctcb_run", False)]:
        root.removeHandler(old)
    sinks = [logging.FileHandler(run.file("train.log" if rank == 0 else "train.%d.log" % rank))]
    if not quiet:
        sinks.append(logging.StreamHandler())
    for h in sinks:
        h._ctcb_run = True
        root.addHandler(h)
    return root


def run(args=None):
    cli = _parse(args)
    rank, world = _select_device()
    resumed = cli.cfg_file is not None
    cfg = run_config(cli)
    cfg.update(host=get_hostname(), git_rev=get_git_revision(), pid=os.getpid(), test=cli.test)

    if resumed:
        out_dir = cfg["output_dir"]
    else:
        # the run directory is named by rank 0's clock and SHARED: ranks started a second apart would otherwise
        # log into (and resume from) directories that do not exist
        out_dir = os.path.join(cli.runDir, str(TimeString()))
        if world > 1:
            import torch.distributed as dist
            box = [out_dir]
            dist.broadcast_object_list(box, src=0)
            out_dir = box[0]
        if rank == 0:
            os.makedirs(out_dir, exist_ok=True)
        cli.cfg_file = os.path.join(out_dir, "cfg.json")
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
    cfg["output_dir"] = out_dir
    cfg["in_file"] = cfg["out_file"] = os.path.join(out_dir, "params.pk")
    if cli.test:                                      # these come from the command line, not the stored config
        for key in ("dataDir", "numFiles", "startFile", "outDir", "maxUtts", "lastWeights"):
            cfg[key] = getattr(cli, key)

    run_dir = RunDir(out_dir)
    log = _attach_logging(run_dir, rank, cfg["quiet"])
    log.info("Running on %s" % cfg["host"])
    np.random.seed(33)                                # runNNet.py:113-115
    random.seed(33)

    opts = CfgStruct(**cfg)
    opts.cfg_file = cli.cfg_file
    if cli.test:
        return test(opts, rank, world)
    return _train(opts, cfg, run_dir, log, rank, world)


def _train(opts, cfg, run_dir, log, rank, world):
    loader = dl.DataLoader(opts.dataDir, opts.rawDim, opts.inputDim, opts.alisDir or opts.dataDir)
    net = rnnet.NNet(opts.inputDim, opts.outputDim, opts.layerSize, opts.numLayers, opts.maxUttLen,
                     temporalLayer=opts.temporalLayer, reg=opts.reg, numTemporal=opts.numTemporal,
                     maxUtts=utterance_capacity(opts, world),
                     maxLabels=min(opts.maxLabels, opts.maxUttLen), dropout=opts.dropout, cell=opts.cell,
                     layerNorm=opts.layerNorm, subsample=opts.subsample, subsampleLayer=opts.subsampleLayer,
                     peephole=opts.peephole, freqMasks=opts.freqMasks, freqMaskWidth=opts.freqMaskWidth,
                     timeMasks=opts.timeMasks, timeMaskWidth=opts.timeMaskWidth, timeMaskRatio=opts.timeMaskRatio,
                     featDim=opts.featDim, weightNoise=opts.weightNoise, zoneoutCell=opts.zoneoutCell,
                     zoneoutHidden=opts.zoneoutHidden, interLayer=opts.interLayer, interWeight=opts.interWeight,
                     selfCondition=opts.selfCondition, tf32=opts.tf32)
    net.initParams()
    optimizer = sgd.SGD(net, opts.maxUttLen, alpha=opts.step, optimizer=opts.optimizer, momentum=opts.momentum,
                        batchSize=opts.batchSize, verbose=(rank == 0 and not opts.quiet), beta1=opts.beta1,
                        beta2=opts.beta2, epsilon=opts.epsilon, emaDecay=opts.emaDecay)
    cfg["param_count"] = net.paramCount()
    if rank == 0:
        dump_config(cfg, opts.cfg_file)

    first_epoch = run_dir.read_int("epoch", -1) + 1
    if os.path.exists(opts.in_file):                  # resume: optimiser state, then the stack (then the average)
        with open(opts.in_file, "rb") as fid:
            optimizer.fromFile(fid)
            optimizer.alpha = optimizer.alpha / (opts.anneal ** first_epoch)
            net.fromFile(fid)
            if optimizer.average is not None:
                optimizer.averageFromFile(fid)

    for epoch in range(first_epoch, opts.epochs):
        order = np.random.permutation(opts.numFiles) + 1
        loader.loadDataFileAsynch(order[0])
        first_file = 0
        if epoch == first_epoch:
            first_file = run_dir.read_int("num_files", 0)
            if first_file:
                log.info("Starting from file %d, epoch %d" % (first_file, first_epoch))
        elif rank == 0:
            run_dir.write("num_files", 0)

        for n in range(first_file, len(order)):
            tic = time.time()
            data_dict, alis, keys, sizes = loader.getDataAsynch()
            if n + 1 < len(order):                    # prefetch the next file while this one trains
                loader.loadDataFileAsynch(order[n + 1])
            optimizer.run(data_dict, alis, keys, sizes)
            log.info("File time %f" % (time.time() - tic))
            if (n + 1) % opts.save_every == 0 and rank == 0:
                log.info("Saving parameters")
                run_dir.checkpoint(optimizer, net)
                run_dir.write("num_files", n + 1)
                if optimizer.expcost:
                    smooth = optimizer.expcost[-1]
                    if opts.reg > 0.0 and optimizer.regcost:
                        smooth -= optimizer.regcost[-1]
                    run_dir.write("last_cost", smooth)

        if rank == 0:
            run_dir.write("epoch", epoch)
            run_dir.checkpoint(optimizer, net, suffix=".epoch{0:02}".format(epoch))
        optimizer.alpha = optimizer.alpha / opts.anneal

    if rank == 0:
        touch_file(run_dir.file("sentinel"))          # run complete
    return optimizer, net


def test(opts, rank=0, world=1):
    """Forward-only pass of a trained model over data files; writes Kaldi arks + pickles
    (runNNet.py:208-237, analysis-utils/writeLikelihoods.py).  --maxUtts utterances per forward call (0: one, the
    reference's loop); rank `rank` of `world` processes (run() passes them under torchrun) writes its own share of
    the files (parallel.rank_files).  A model trained with --emaDecay writes the arks from its weight average (the
    third pickle of params.pk), or from its last weights with --lastWeights."""
    trained = trained_config(opts.cfg_file)
    logging.getLogger().info("Running on %s" % get_hostname())
    # the intermediate CTC loss only trains, unless the net conditions its upper layers on it
    cond = dict(interLayer=trained.interLayer, interWeight=trained.interWeight,
                selfCondition=True) if trained.selfCondition else {}
    net = rnnet.NNet(trained.inputDim, trained.outputDim, trained.layerSize, trained.numLayers, trained.maxUttLen,
                     temporalLayer=trained.temporalLayer, train=False, maxUtts=max(1, opts.maxUtts),
                     numTemporal=trained.numTemporal, cell=trained.cell, layerNorm=trained.layerNorm,
                     subsample=trained.subsample, subsampleLayer=trained.subsampleLayer, peephole=trained.peephole,
                     zoneoutCell=trained.zoneoutCell, zoneoutHidden=trained.zoneoutHidden, tf32=trained.tf32, **cond)
    net.initParams()
    with open(trained.in_file, "rb") as fid:
        pickle.load(fid)                              # optimiser state: not needed here
        net.fromFile(fid)
        if trained.emaDecay > 0.0 and not getattr(opts, "lastWeights", False):
            net.fromFile(fid)                         # the average, in the stack's format
    loader = dl.DataLoader(opts.dataDir, trained.rawDim, trained.inputDim, opts.alisDir or opts.dataDir)
    out_dir = getattr(opts, "outDir", None) or os.path.join(opts.output_dir, "ctc_loglikes")
    os.makedirs(out_dir, exist_ok=True)
    for filenum in parallel.rank_files(opts.startFile, opts.numFiles, rank, world):
        writeLogLikes(loader, net, filenum, out_dir, writePickle=True)
    return net


if __name__ == "__main__":
    run()
