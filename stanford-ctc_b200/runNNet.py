"""runNNet -- training / likelihood-dump driver for the H100 backend.

Call surface kept from the reference driver (ctc_fast/runNNet.py:23-237): `run(args)` and
`test(opts)`, every command-line flag of runNNet.py:27-69 with its default, the run-directory protocol
(cfg.json, params.pk = SGD pickle followed by the stack pickle, params.pk.epochNN, epoch, num_files,
last_cost, sentinel, train.log), resume through --cfg_file with the step size re-annealed
(runNNet.py:143-166), the fixed seeds 33 (:113-115) and CUDA_DEVICE device selection (:117-120).
The implementation is organised differently: a declarative flag table, one RunDir helper that owns the
side files, and separate train/evaluate phases.  Site paths of run_cfg.py / decoder_config.py became
flags (--runDir, --outDir); new flags: --numTemporal, --batchSize, --maxUtts, --maxLabels, --quiet.  Under torchrun the same
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
    ("batchSize", int, 1, "utterances per optimisation step (1 = the reference schedule)"),
    ("maxUtts", int, 0, "utterances per micro-batch per GPU: a larger shard accumulates its gradient over several "
                        "micro-batches (0 = the whole shard, batchSize / number of GPUs rounded up); with --test, "
                        "utterances per forward call per GPU (0 = one, the reference's loop)"),
    ("maxLabels", int, 511, "longest label sequence the buffers are sized for"),
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
        with open(self.file("params.pk") + suffix, "wb") as fid:     # two pickles back to back
            optimizer.toFile(fid)
            net.toFile(fid)


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
        for key in ("dataDir", "numFiles", "startFile", "outDir", "maxUtts"):
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
                     maxLabels=min(opts.maxLabels, opts.maxUttLen))
    net.initParams()
    optimizer = sgd.SGD(net, opts.maxUttLen, alpha=opts.step, momentum=opts.momentum, batchSize=opts.batchSize,
                        verbose=(rank == 0 and not opts.quiet))
    cfg["param_count"] = net.paramCount()
    if rank == 0:
        dump_config(cfg, opts.cfg_file)

    first_epoch = run_dir.read_int("epoch", -1) + 1
    if os.path.exists(opts.in_file):                  # resume: optimiser state, then the stack
        with open(opts.in_file, "rb") as fid:
            optimizer.fromFile(fid)
            optimizer.alpha = optimizer.alpha / (opts.anneal ** first_epoch)
            net.fromFile(fid)

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
    the files (parallel.rank_files)."""
    trained = trained_config(opts.cfg_file)
    logging.getLogger().info("Running on %s" % get_hostname())
    net = rnnet.NNet(trained.inputDim, trained.outputDim, trained.layerSize, trained.numLayers, trained.maxUttLen,
                     temporalLayer=trained.temporalLayer, train=False, maxUtts=max(1, opts.maxUtts),
                     numTemporal=trained.numTemporal)
    net.initParams()
    with open(trained.in_file, "rb") as fid:
        pickle.load(fid)                              # optimiser state: not needed here
        net.fromFile(fid)
    loader = dl.DataLoader(opts.dataDir, trained.rawDim, trained.inputDim, opts.alisDir or opts.dataDir)
    out_dir = getattr(opts, "outDir", None) or os.path.join(opts.output_dir, "ctc_loglikes")
    os.makedirs(out_dir, exist_ok=True)
    for filenum in parallel.rank_files(opts.startFile, opts.numFiles, rank, world):
        writeLogLikes(loader, net, filenum, out_dir, writePickle=True)
    return net


if __name__ == "__main__":
    run()
