"""CPU tests of TF32 mode (ctcb_brnn_config.tf32): the config contract, workspaces that do not depend on the mode, and
the Python and runNNet surface."""
import ctypes
import inspect

import config_matrix


def _cfg(**kw):
    import _ctcb
    cfg = _ctcb.BrnnConfig(41 * 15, 11, 1024, 3, 2, 60, 8, 20, 0.0, 20.0, 0, 1, 0)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def test_config_refusals():
    from _ctcb import lib
    assert _cfg().tf32 == 0               # an initialiser without the member keeps its meaning
    for bad in (2, -1, 7):
        cfg = _cfg(tf32=bad)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0, bad
        assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) == 0, bad
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1, bad
        assert b"tf32 %d is neither 0" % bad in lib.ctcb_last_error(), lib.ctcb_last_error()
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(_cfg(tf32=1)), ctypes.byref(h)) == 0, lib.ctcb_last_error()
    lib.ctcb_brnn_destroy(h)


def test_every_config_answer_is_the_same_in_both_modes():
    """Parameter layout, both workspace sizes, the error-flag offsets, every activation offset and create's answer, over
    the whole config matrix: TF32 mode moves nothing."""
    import _ctcb
    lib = config_matrix.bind(_ctcb.lib, _ctcb.BrnnConfig)
    for entry in config_matrix.MATRIX:
        off = config_matrix.config(_ctcb.BrnnConfig, entry)
        on = config_matrix.config(_ctcb.BrnnConfig, entry)
        on.tf32 = 1
        assert config_matrix.answers(lib, on) == config_matrix.answers(lib, off), entry


def test_standalone_entry_points_share_the_workspace_of_the_default():
    """The TF32 entry points take the same arguments and workspace sizes as the default ones."""
    import _ctcb
    P = _ctcb._PROTOS
    for name in ("ctcb_gemm", "ctcb_gemm_pair", "ctcb_brnn_sweep"):
        assert P[name + "_tf32"] == P[name + "_f32"], name
    for name in ("ctcb_debug_gemm_plan", "ctcb_debug_sweep_plan"):
        assert P[name + "_tf32"] == P[name], name


def test_nnet_flag_defaults_off():
    import nnets.brnnet
    import nnets.nnet
    import nnets.rnnet
    for cls in (nnets.brnnet.NNet, nnets.rnnet.NNet, nnets.nnet.NNet):
        assert inspect.signature(cls.__init__).parameters["tf32"].default is False, cls


def test_runnnet_tf32_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    assert runNNet._parse([]).tf32 is False
    assert any(f[0] == "tf32" and f[1] is None and f[3] for f in runNNet.FLAGS)
    cfg = runNNet.run_config(runNNet._parse(["--tf32"]))
    assert cfg["tf32"] is True
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["tf32"] is True
    assert runNNet.trained_config(f).tf32 is True
    old = {k: v for k, v in cfg.items() if k != "tf32"}
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["tf32"] is False
    assert runNNet.trained_config(f2).tf32 is False

