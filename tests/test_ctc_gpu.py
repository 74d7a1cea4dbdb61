"""GPU parity tests of the CTC kernel, through the C ABI (ctcb_ctc_loss_grad_f32) and the drop-in
module ctc_fast, against (a) the committed golden vectors produced by the unmodified reference
ctc_fast.pyx and (b) the oracle run live on the same inputs.

Tolerance (BASELINE.json north_star / SURVEY.md 8c): |nll - ref| / |ref| <= 1e-4 and
||g - g_ref||_F / ||g_ref||_F <= 1e-4 in fp32, skip flags equal."""
import functools

import numpy as np
import pytest

import recipes
from oracle import ctc_oracle
from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
TOL = 1e-4
_forced = None             # the organisation _run_forced has set with CTCB_CTC, None: automatic


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


def _gpu_single(torch, probs, seq, is_prob=True):
    """One utterance through ctc_loss_batch in [B][T][K] layout; probs is K x T."""
    import ctc_fast
    K, T = probs.shape
    acts = torch.from_numpy(np.ascontiguousarray(probs.T, dtype=np.float32)).cuda().view(1, T, K)
    lab = torch.from_numpy(seq if seq.size else np.zeros(1, np.int32)).cuda()
    off = torch.tensor([0, seq.shape[0]], dtype=torch.int32).cuda()
    tl = torch.tensor([T], dtype=torch.int32).cuda()
    if _forced == "ckpt" and seq.shape[0] > 127:
        # the checkpoint kernel has no build beyond 127 labels: forced, the call is an error, never another kernel
        with pytest.raises(ValueError, match="ckpt"):
            ctc_fast.ctc_loss_batch(acts, tl, lab, off, seq.shape[0], is_prob=is_prob)
        pytest.skip("CTCB_CTC=ckpt refuses %d labels" % seq.shape[0])
    nll, grad, skip = ctc_fast.ctc_loss_batch(acts, tl, lab, off, seq.shape[0], is_prob=is_prob)
    return float(nll.item()), grad.view(T, K).cpu().numpy().T.astype(np.float64), bool(skip.item())


@pytest.mark.parametrize("name", recipes.ALL_CTC)
def test_golden_cases_through_c_abi(name, golden_ctc, cuda):
    probs, seq = recipes.ctc_case(name)
    nll, grad, skip = _gpu_single(cuda, probs, seq)
    assert skip == bool(golden_ctc[name + "/skip"])
    if skip:
        assert not grad.any()
        return
    g_nll = float(golden_ctc[name + "/nll"])
    st = recipes.golden_stride(*probs.shape)
    if np.isinf(g_nll):
        assert np.isinf(nll) and nll > 0
    else:
        assert abs(nll - g_nll) / abs(g_nll) <= TOL
    assert _rel(grad[:, ::st], golden_ctc[name + "/grad"].astype(np.float64)) <= TOL


@pytest.mark.parametrize("name", ["c1", "ctc_py", "repeat_heavy", "T_equals_L", "single_label"])
def test_dropin_ctc_loss_signature_and_parity(name, cuda):
    """ctc_fast.ctc_loss(params, seq, blank=0): reference argument/return contract."""
    import ctc_fast
    probs, seq = recipes.ctc_case(name)
    P = np.asfortranarray(probs.astype(np.float64))
    nll, grad, skip = ctc_fast.ctc_loss(P, seq)
    o_nll, o_grad, o_skip = ctc_oracle.ctc_loss(P, seq)
    assert isinstance(nll, float) and isinstance(skip, bool)
    assert grad.dtype == np.float64 and grad.shape == P.shape and grad.flags.f_contiguous
    assert skip == o_skip
    if not skip:
        assert abs(nll - o_nll) / abs(o_nll) <= TOL and _rel(grad, o_grad) <= TOL
    with pytest.raises(ValueError):
        ctc_fast.ctc_loss(np.ascontiguousarray(P), seq)
    with pytest.raises(ValueError):
        ctc_fast.ctc_loss(P.astype(np.float32), seq)


def test_fused_softmax_logits_path(cuda):
    """is_prob=0: logits in, softmax fused (the brnnet.py:161-175 path)."""
    logits, seq = recipes.synth_ctc(300, 62, 40, seed=5)
    probs = recipes.softmax_cols(logits.astype(np.float32).astype(np.float64)).astype(np.float32)
    nll, grad, skip = _gpu_single(cuda, logits.astype(np.float32), seq, is_prob=False)
    o_nll, o_grad, o_skip = ctc_oracle.ctc_loss(np.asfortranarray(probs.astype(np.float64)), seq)
    assert not skip and not o_skip
    assert abs(nll - o_nll) / abs(o_nll) <= TOL and _rel(grad, o_grad) <= TOL


def test_ragged_batch_time_major_layout(cuda):
    """B utterances of different lengths in the time-major [Tmax][B][K] layout the BRNN uses;
    includes an infeasible utterance (skip), a too-short one (inf) and an empty tail."""
    import ctc_fast
    torch = cuda
    K = 35
    lens = [90, 64, 7, 33, 90, 5, 48, 12, 77]
    nlabs = [20, 10, 7, 33, 1, 9, 15, 3, 30]
    rng = np.random.RandomState(12)
    B, Tmax = len(lens), max(lens)
    logits = rng.randn(Tmax, B, K).astype(np.float32) * 2.0
    seqs = [(1 + rng.randint(0, K - 1, size=n)).astype(np.int32) for n in nlabs]
    seqs[2] = np.array([3, 3, 3, 3, 5, 5, 6], dtype=np.int32)   # T == |l| with repeats: infeasible -> skip
    off = np.concatenate([[0], np.cumsum(nlabs)]).astype(np.int32)
    acts = torch.from_numpy(logits).cuda()
    nll, grad, skip = ctc_fast.ctc_loss_batch(
        acts, torch.tensor(lens, dtype=torch.int32).cuda(), torch.from_numpy(np.concatenate(seqs)).cuda(),
        torch.from_numpy(off).cuda(), max(nlabs), is_prob=False, utt_stride=K, frame_stride=B * K)
    nll, grad, skip = nll.cpu().numpy(), grad.cpu().numpy(), skip.cpu().numpy()
    for u in range(B):
        T = lens[u]
        p = recipes.softmax_cols(logits[:T, u, :].T.astype(np.float64)).astype(np.float32)
        o_nll, o_grad, o_skip = ctc_oracle.ctc_loss(np.asfortranarray(p.astype(np.float64)), seqs[u])
        assert bool(skip[u]) == o_skip, u
        assert not grad[T:, u, :].any()                 # padded frames carry no gradient
        if o_skip:
            assert not grad[:, u, :].any()
        elif np.isinf(o_nll):
            assert np.isinf(nll[u]) and _rel(grad[:T, u, :].T, o_grad) <= TOL
        else:
            assert abs(nll[u] - o_nll) / abs(o_nll) <= TOL, u
            assert _rel(grad[:T, u, :].T.astype(np.float64), o_grad) <= TOL, u


PAIRS_PER_LANE_NLAB = [31, 32, 63, 64, 127, 128, 255, 256, 400, 511]


@pytest.mark.parametrize("nlab", PAIRS_PER_LANE_NLAB)
def test_pairs_per_lane_boundaries(nlab, cuda):
    """Label counts around every register-tiling boundary (1,2,4,8,16 pairs per lane)."""
    T = nlab + 40
    logits, seq = recipes.synth_ctc(T, 20, nlab, seed=nlab)
    probs = recipes.softmax_cols(logits).astype(np.float32)
    nll, grad, skip = _gpu_single(cuda, probs, seq)
    o_nll, o_grad, o_skip = ctc_oracle.ctc_loss(np.asfortranarray(probs.astype(np.float64)), seq)
    assert skip == o_skip
    if not skip:
        assert abs(nll - o_nll) / abs(o_nll) <= TOL and _rel(grad, o_grad) <= TOL


def test_too_many_labels_is_an_error_not_a_fallback(cuda):
    logits, seq = recipes.synth_ctc(700, 20, 600, seed=1)
    with pytest.raises((ValueError, MemoryError)):
        _gpu_single(cuda, recipes.softmax_cols(logits).astype(np.float32), seq)


def test_full_size_properties(cuda):
    """BASELINE-size batch (TIMIT shape x 4096 utterances, > L2): size-independent properties --
    every gradient frame sums to 0 (softmax minus a distribution), nll > 0 and finite, identical
    utterances give identical results, and a spot-checked subset matches the oracle."""
    import ctc_fast
    torch = cuda
    B, T, K, nlab = 4096, 200, 62, 30
    g = torch.Generator(device="cuda").manual_seed(3)
    acts = torch.randn(B, T, K, device="cuda", generator=g)
    acts[B - 1] = acts[0]
    rng = np.random.RandomState(4)
    seqs = (1 + rng.randint(0, K - 1, size=(B, nlab))).astype(np.int32)
    seqs[B - 1] = seqs[0]
    nll, grad, skip = ctc_fast.ctc_loss_batch(
        acts, torch.full((B,), T, dtype=torch.int32, device="cuda"), torch.from_numpy(seqs.ravel()).cuda(),
        torch.arange(0, (B + 1) * nlab, nlab, dtype=torch.int32, device="cuda"), nlab, is_prob=False)
    assert int(skip.sum()) == 0
    assert bool(torch.isfinite(nll).all()) and float(nll.min()) > 0
    assert float(grad.sum(dim=2).abs().max()) < 2e-5
    assert float((nll[0] - nll[B - 1]).abs()) == 0.0 and bool((grad[0] == grad[B - 1]).all())
    for u in (0, 1777, 4094):
        p = recipes.softmax_cols(acts[u].cpu().numpy().T.astype(np.float64)).astype(np.float32)
        o_nll, o_grad, _ = ctc_oracle.ctc_loss(np.asfortranarray(p.astype(np.float64)), seqs[u])
        assert abs(float(nll[u]) - o_nll) / o_nll <= TOL
        assert _rel(grad[u].cpu().numpy().T.astype(np.float64), o_grad) <= TOL


def test_best_path_matches_reference_semantics(cuda):
    import ctc_fast
    probs, _ = recipes.ctc_case("time_trials")
    P = np.asfortranarray(probs.astype(np.float64))
    hyp, align = ctc_fast.decode_best_path(P)
    o_hyp, o_align = ctc_oracle.decode_best_path(P)
    assert hyp == o_hyp and align == o_align
    q = np.zeros((10, 9)); q[[0, 3, 3, 0, 3, 1, 5, 5, 8], np.arange(9)] = 1.0
    assert ctc_fast.decode_best_path(np.asfortranarray(q)) == ([3, 3, 5], [2, 4, 7])


def _run_forced(shape, knobs, golden_ctc, torch):
    """The golden / edge cases of this file in this process with CTCB_CTC=shape; returns the reasons of those that
    skipped."""
    global _forced
    cases = ([functools.partial(test_golden_cases_through_c_abi, n, golden_ctc) for n in recipes.ALL_CTC]
             + [test_ragged_batch_time_major_layout]
             + [functools.partial(test_pairs_per_lane_boundaries, n) for n in PAIRS_PER_LANE_NLAB]
             + [test_fused_softmax_logits_path]
             + [functools.partial(test_meet_in_the_middle_tile_boundaries, T) for T in TILE_BOUNDARY_T]
             + [test_full_size_properties])
    knobs("CTCB_CTC", shape)
    _forced = shape
    skipped = []
    try:
        for case in cases:
            try:
                case(torch)
            except pytest.skip.Exception as e:
                skipped.append(str(e))
    finally:
        _forced = None
    return skipped


@pytest.mark.parametrize("shape", ["warp", "pair"])
def test_other_kernel_shapes_when_forced(shape, knobs, golden_ctc, cuda):
    """Small batches take the three-phase latency kernel (recurrences on two warps, gradient on all warps); CTCB_CTC=warp
    forces the one-warp-per-utterance kernel that spills the trellis (large batches, long label sequences), CTCB_CTC=pair
    the two-warp meet-in-the-middle kernel (mid-sized batches), through the same golden / edge cases."""
    skipped = _run_forced(shape, knobs, golden_ctc, cuda)
    assert not skipped, skipped


def test_checkpoint_kernel_when_forced(knobs, golden_ctc, cuda):
    """CTCB_CTC=ckpt forces the one-warp kernel that checkpoints the trellis and recomputes it on chip (large batches) through
    the same golden / edge cases.  It has no build beyond 127 labels: those cases must be refused with CTCB_EINVAL, never
    run on another kernel."""
    skipped = _run_forced("ckpt", knobs, golden_ctc, cuda)
    # 3 golden cases and 5 label counts have more than 127 labels; each is skipped after its refusal was checked
    assert len(skipped) == 8 and all("CTCB_CTC=ckpt refuses" in s for s in skipped), skipped


TILE_BOUNDARY_T = [1, 3, 7, 8, 9, 16, 17, 31, 32, 33, 47, 200]


@pytest.mark.parametrize("T", TILE_BOUNDARY_T)
def test_meet_in_the_middle_tile_boundaries(T, cuda):
    """Utterance lengths around the tile sizes (16 frames; 8 in the checkpoint kernel): 1 tile (no first half), odd/even
    tile counts."""
    rng = np.random.RandomState(100 + T)
    K = 20
    nlab = max(1, min(T // 2, 6))
    logits = rng.randn(K, T)
    seq = (1 + rng.randint(0, K - 1, size=nlab)).astype(np.int32)
    probs = recipes.softmax_cols(logits).astype(np.float32)
    nll, grad, skip = _gpu_single(cuda, probs, seq)
    o_nll, o_grad, o_skip = ctc_oracle.ctc_loss(np.asfortranarray(probs.astype(np.float64)), seq)
    assert skip == o_skip
    if not skip:
        assert abs(nll - o_nll) / abs(o_nll) <= TOL
        assert _rel(grad, o_grad) <= TOL
