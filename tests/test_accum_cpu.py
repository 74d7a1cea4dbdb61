"""CPU tests of gradient accumulation's host side: how a rank's shard of a step is cut into micro-batches
(parallel.micro_batches), how many utterances a micro-batch holds (parallel.micro_batch_capacity), and the
runNNet flag --maxUtts that sets it (parsed, stored in cfg.json, honoured on resume)."""
import itertools
import os

import pytest


def test_micro_batches_cover_every_utterance_once_in_order():
    import parallel
    for n, cap in itertools.product(range(0, 23), range(1, 9)):
        utts = ["u%d" % i for i in range(n)]
        pieces = parallel.micro_batches(utts, cap)
        assert [u for p in pieces for u in p] == utts                 # coverage, each once, order kept
        assert all(1 <= len(p) <= cap for p in pieces)                # the cap, and no empty piece
        assert len(pieces) == -(-n // cap)                            # as few pieces as the cap allows
        assert all(len(p) == cap for p in pieces[:-1])                # only the last one may be short


def test_micro_batches_examples_and_edge_cases():
    import parallel
    assert parallel.micro_batches([], 3) == []
    assert parallel.micro_batches(range(8), 3) == [[0, 1, 2], [3, 4, 5], [6, 7]]
    assert parallel.micro_batches(range(8), 8) == [list(range(8))]
    assert parallel.micro_batches(range(3), 10) == [[0, 1, 2]]
    assert parallel.micro_batches(iter("abcde"), 2) == [["a", "b"], ["c", "d"], ["e"]]
    with pytest.raises(ValueError):
        parallel.micro_batches([1, 2], 0)


def test_micro_batches_of_every_rank_cover_the_step():
    """Sharded first, then cut: every admitted utterance is computed exactly once over all ranks' micro-batches,
    and no rank needs more than one micro-batch more than another."""
    import parallel
    items = list(range(7))
    for world, cap in ((1, 3), (2, 2), (3, 1), (4, 2)):
        per_rank = [parallel.micro_batches(parallel.shard(items, r, world), cap) for r in range(world)]
        assert sorted(u for ps in per_rank for p in ps for u in p) == items
        counts = [len(ps) for ps in per_rank]
        assert max(counts) - min(counts) <= 1


def test_micro_batch_capacity_default_is_the_whole_shard():
    import parallel
    for bs, world in itertools.product((1, 5, 7, 8, 256), (1, 2, 3, 8)):
        assert parallel.micro_batch_capacity(0, bs, world) == parallel.per_rank_capacity(bs, world)
        assert parallel.micro_batch_capacity(2, bs, world) == min(2, parallel.per_rank_capacity(bs, world))
    assert parallel.micro_batch_capacity(32, 256, 1) == 32
    assert parallel.micro_batch_capacity(500, 256, 2) == 128     # never more than a shard holds


def test_runnnet_max_utts_flag_is_parsed_stored_and_kept_on_resume(tmp_path):
    import runNNet
    from run_utils import dump_config, load_config, CfgStruct
    cli = runNNet._parse([])
    assert cli.maxUtts == 0
    cfg = runNNet.run_config(cli)
    assert cfg["maxUtts"] == 0
    assert runNNet.utterance_capacity(CfgStruct(**cfg), 1) == 1                  # batchSize 1, one GPU
    opts = CfgStruct(**runNNet.run_config(runNNet._parse(["--batchSize", "7"])))
    assert runNNet.utterance_capacity(opts, 2) == 4                               # today's per_rank_capacity(7, 2)

    cli = runNNet._parse(["--batchSize", "256", "--maxUtts", "32"])
    assert cli.maxUtts == 32
    cfg = runNNet.run_config(cli)
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert load_config(f)["maxUtts"] == 32
    # resume: the stored configuration wins over the command line's defaults
    resumed = runNNet.run_config(runNNet._parse(["--cfg_file", f]))
    assert resumed["maxUtts"] == 32 and resumed["batchSize"] == 256
    assert runNNet.utterance_capacity(CfgStruct(**resumed), 1) == 32
    assert runNNet.utterance_capacity(CfgStruct(**resumed), 4) == 32
    # a run recorded before the flag existed resumes with the whole-shard default
    old = dict(cfg)
    del old["maxUtts"]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    resumed_old = runNNet.run_config(runNNet._parse(["--cfg_file", f2]))
    assert resumed_old["maxUtts"] == 0
    assert runNNet.utterance_capacity(CfgStruct(**resumed_old), 2) == 128


def test_part_flags_match_the_header():
    import re
    import _ctcb
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "include", "ctcb200.h")).read()
    first = int(re.search(r"#define CTCB_PART_FIRST (\d+)", src).group(1))
    last = int(re.search(r"#define CTCB_PART_LAST (\d+)", src).group(1))
    assert (_ctcb.PART_FIRST, _ctcb.PART_LAST) == (first, last) and first & last == 0
