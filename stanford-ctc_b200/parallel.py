"""parallel -- host-side logic of the data-parallel step (pure Python, no CUDA).

The reference has no multi-GPU training (one process, one GPU, one utterance per step:
ctc_fast/runNNet.py:117-120, sgd.py:70-95).  Utterances are independent until the
parameter update, so a step's minibatch is sharded over ranks and the flat gradient (with its
4-float statistics tail) is summed by ONE all-reduce; every rank then applies the identical update.
"""


def shard(items, rank, world):
    """Round-robin shard of one step's utterances: rank r takes items r, r+world, ...  Every item is
    owned by exactly one rank and the per-rank counts differ by at most one."""
    if world <= 1:
        return list(items)
    return list(items[rank::world])


def select_step_utterances(data_dict, alis, chunk, max_frames, rank, world, log=None, max_labels=None):
    """The utterances of one step that THIS rank computes.  The reference's per-utterance admission rules
    (sgd.py:76-88: skip when longer than the buffers, skip when there are fewer frames than labels) are applied
    to the whole step in the same order on every rank -- two cheap length look-ups per key -- and only then is
    the list sharded, so all ranks agree on the shards without looking at each other's data."""
    used = []
    for k in chunk:
        nframes = data_dict[k].shape[1]
        if nframes > max_frames:
            if log:
                log("SKIPPING utt exceeds batch length (Utterance length %d)." % nframes)
            continue
        nlab = len(alis[k])
        if nframes < nlab:
            if log:
                log("SKIPPING utt frames less than label length (Utterance length %d, Num Labels %d)." % (nframes, nlab))
            continue
        if max_labels is not None and nlab > max_labels:
            # not a reference rule: the device buffers (and the CTC kernel) hold at most max_labels labels per utterance
            if log:
                log("SKIPPING utt label sequence exceeds the label capacity (Num Labels %d, capacity %d)." % (nlab, max_labels))
            continue
        used.append(k)
    return shard(used, rank, world)


def bucketed_chunks(keys, length_of, batch_size, pool_batches=16, rng=None):
    """Minibatches of similar length from an already shuffled key list (SURVEY.md 8f-2; the reference steps one
    utterance at a time, sgd.py:68-70, so it never pads).  The shuffled list is cut into pools of
    pool_batches * batch_size keys; each pool is sorted by length and cut into minibatches, and the minibatches of a
    pool are visited in random order -- every key is used exactly once per call, the padding of a step drops from
    max/mean over the corpus to max/mean over ~1/pool_batches of it.  batch_size == 1 returns the shuffled order
    unchanged (the reference's schedule).  Returns (chunks, padded_frames, real_frames)."""
    if batch_size <= 1:
        ks = list(keys)
        n = sum(length_of(k) for k in ks)
        return [[k] for k in ks], n, n
    import random as _random
    rng = rng or _random
    chunks, padded, real = [], 0, 0
    pool = max(1, pool_batches) * batch_size
    for p0 in range(0, len(keys), pool):
        part = sorted(keys[p0:p0 + pool], key=length_of)
        cs = [part[i:i + batch_size] for i in range(0, len(part), batch_size)]
        rng.shuffle(cs)
        for c in cs:
            ls = [length_of(k) for k in c]
            padded += max(ls) * len(ls)
            real += sum(ls)
        chunks.extend(cs)
    return chunks, padded, real


def per_rank_capacity(batch_size, world):
    """Utterance capacity each rank must allocate for a global step of batch_size utterances."""
    return (batch_size + world - 1) // max(world, 1)


def world_info():
    """(dist module or None, rank, world) from torch.distributed if it is initialised."""
    try:
        import torch.distributed as dist
    except Exception:
        return None, 0, 1
    if dist.is_available() and dist.is_initialized():
        return dist, dist.get_rank(), dist.get_world_size()
    return None, 0, 1


def allreduce_sum(dist, flat):
    """Sum the flat gradient (+ statistics tail) over ranks, in place."""
    if dist is not None:
        dist.all_reduce(flat)
    return flat
