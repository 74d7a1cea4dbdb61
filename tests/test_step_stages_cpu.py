"""CPU tests of the activation hook's entries for the stage checks of test_step_stages_gpu.py: what = 15..17 (z, Mu and
Rstd of a layer-normalised layer), 18 (the masked feature copy) and 19 (the noisy parameter copy).  Each lies inside
the training workspace, 256-byte aligned, at the width the header gives, overlaps no other entry of the hook, and is
refused (CTCB_EINVAL) where its feature is off.  The hook adds no buffer: the training and forward-only workspace sizes
are pinned below at those of the layout before these entries existed."""
import ctypes

import pytest

H, T, B = 64, 60, 8


def _cfg(**kw):
    import _ctcb
    cfg = _ctcb.BrnnConfig(41 * 15, 11, H, 3, 2, T, B, 20, 0.0, 20.0, 0, 1, 0)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


# name: (config, the layer-normalised layers, (training, forward-only) workspace bytes of the layout)
CASES = {
    "plain": (dict(), [], (2953472, 1078272)),
    "ln": (dict(layerNorm=1), [1, 3], (3238144, 1078272)),
    "ln_dnn": (dict(layerNorm=1, temporalLayer=0), [1, 2, 3], (2782464, 741376)),
    "ln_sub_above": (dict(layerNorm=1, subsample=2, subsampleLayer=3), [1, 3], (2979840, 1201408)),
    "ln_masks_noise": (dict(layerNorm=1, maskFeatDim=41, weightNoise=1), [1, 3], (4646912, 1078272)),
    "masks": (dict(maskFeatDim=41), [], (4134400, 1078272)),
    "noise": (dict(weightNoise=1), [], (3180288, 1078272)),
    "lstm_noise_cond": (dict(cell=1, weightNoise=1, interLayer=1, interWeight=0.3, selfCondition=1), [],
                        (5622784, 3122688)),
}


def _hook(cfg, what, layer):
    from _ctcb import lib
    off, width = ctypes.c_size_t(), ctypes.c_int32()
    rc = lib.ctcb_brnn_activation_offset(ctypes.byref(cfg), what, layer, ctypes.byref(off), ctypes.byref(width))
    return None if rc else (off.value, width.value)


def _rows(cfg, i):
    """Rows of layer i's buffers at maxT x maxB: the reduced rate from the subsampling layer up."""
    k = cfg.subsample if cfg.subsample >= 2 else 1
    return (-(-T // k) if k > 1 and i >= cfg.subsampleLayer else T) * B


def _entries(cfg):
    """{(what, layer): (offset, bytes)} of every entry the hook gives for cfg, each at the rows of its layer at maxT x
    maxB (what 10 and 11: one float per utterance)."""
    out = {}
    for what in range(20):
        for layer in range(0, cfg.numLayers + 2):
            h = _hook(cfg, what, layer)
            if h is None:
                continue
            off, width = h
            if what == 19:
                n = width
            elif what == 18:
                n = T * B * width
            elif what in (10, 11):
                n = B
            elif 8 <= what <= 14:
                n = _rows(cfg, cfg.interLayer) * width
            else:
                n = _rows(cfg, layer if what in (0, 7) or what >= 15 else cfg.subsampleLayer if what == 6
                          else cfg.temporalLayer) * width
            out[(what, layer)] = (off, 4 * n)
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_offsets_widths_and_refusals(name):
    from _ctcb import lib
    kw, normed, _ = CASES[name]
    cfg = _cfg(**kw)
    total = lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg))
    for layer in range(-1, cfg.numLayers + 3):
        for what in (15, 16, 17):
            h = _hook(cfg, what, layer)
            if layer not in normed:
                assert h is None, (what, layer)
                continue
            off, width = h
            assert width == (H if what == 15 else 1), (what, layer, width)
            assert off % 256 == 0 and off + 4 * _rows(cfg, layer) * width <= total, (what, layer)
    masked, noisy = _hook(cfg, 18, 0), _hook(cfg, 19, 0)
    assert (masked is None) == (cfg.maskFeatDim <= 0)
    assert (noisy is None) == (cfg.weightNoise != 1)
    if masked:
        assert masked[1] == cfg.inputDim and masked[0] % 256 == 0
        assert masked[0] + 4 * T * B * cfg.inputDim <= total
        assert _hook(cfg, 18, 2) == masked            # `layer` is ignored
    if noisy:
        assert noisy[1] == lib.ctcb_brnn_param_count(ctypes.byref(cfg)) and noisy[0] % 256 == 0
        assert noisy[0] + 4 * noisy[1] <= total
        assert _hook(cfg, 19, 3) == noisy
    # a new entry overlaps no other entry of the hook
    ents = _entries(cfg)
    for ka, (oa, na) in ents.items():
        if ka[0] < 15:
            continue
        for kb, (ob, nb) in ents.items():
            if kb != ka and not (ka[0] == kb[0] and oa == ob):
                assert oa + na <= ob or ob + nb <= oa, (ka, kb)


@pytest.mark.parametrize("name", list(CASES))
def test_workspace_sizes_and_other_entries_unchanged(name):
    """The training and forward-only workspace sizes are those of the layout before the hook had these entries, and
    the masked and noisy copies move no layer-normalised layer's entries."""
    from _ctcb import lib
    kw, _, (train_bytes, fwd_bytes) = CASES[name]
    cfg = _cfg(**kw)
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == train_bytes
    assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) == fwd_bytes
    if cfg.maskFeatDim > 0 and cfg.weightNoise == 1:
        ln_only = _cfg(layerNorm=1)
        for layer in (1, 3):
            for what in (15, 16, 17):
                assert _hook(cfg, what, layer) == _hook(ln_only, what, layer)
