"""CPU: the autograd seam's argument checks (b2cnn_train_forward / b2cnn_train_backward / b2cnn_train_step_weighted reject
bad calls before any CUDA call) and the host-side contract of B200TrainableMyCNN and B200Trainer(pos_weight=...)."""
import ctypes

import pytest
import torch

import tskd_b200
from tskd_b200 import capi
from tskd_b200.arch import BLOB_KEYS, ArchConfig
from tskd_b200.trainer import B200Trainer


def _cfg():
    return capi.make_config(tskd_b200.ARCH_PRESETS["mycnn5"])


def _fwd(lib, cfg, mode=capi.MODE_SEQUENCE, ptr=1, ws_bytes=1 << 30):
    p = ctypes.c_void_p(ptr) if ptr else None
    return lib.b2cnn_train_forward(cfg, p, p, 4, p, mode, None, None, p, p, ws_bytes, None)


def _bwd(lib, cfg, mode=capi.MODE_SEQUENCE, ptr=1, ws_bytes=1 << 30):
    p = ctypes.c_void_p(ptr) if ptr else None
    return lib.b2cnn_train_backward(cfg, p, p, 4, p, mode, None, None, p, p, None, None, p, ws_bytes, None)


@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_autograd_entry_points_reject_bad_arguments_before_cuda(call):
    lib = capi.load_library()
    cfg = _cfg()
    assert call(lib, None) == capi.EINVAL
    assert call(lib, ctypes.byref(cfg), ptr=0) == capi.EINVAL and "null" in capi.last_error()
    assert call(lib, ctypes.byref(cfg), mode=7) == capi.EINVAL and "mode" in capi.last_error()
    need = lib.b2cnn_train_workspace_bytes(ctypes.byref(cfg), 4)
    assert call(lib, ctypes.byref(cfg), ws_bytes=need - 1) == capi.ESTATE and "workspace" in capi.last_error()
    relu = capi.make_config(ArchConfig(act="relu"))
    assert call(lib, ctypes.byref(relu)) == capi.EINVAL and "tanh" in capi.last_error()


def test_weighted_step_rejects_bad_arguments_before_cuda():
    lib = capi.load_library()
    cfg = _cfg()
    opt = capi.Adam(1e-5, 0.9, 0.999, 1e-8)
    p = ctypes.c_void_p(1)
    need = lib.b2cnn_train_workspace_bytes(ctypes.byref(cfg), 4)

    def step(pw=13.5, mode=capi.MODE_SEQUENCE, ptr=p, ws=need, o=ctypes.byref(opt)):
        return lib.b2cnn_train_step_weighted(ctypes.byref(cfg), ptr, ptr, ptr, ptr, 1, o, 1, ptr, 4, ptr, ptr, pw, mode, None, None,
                                             ptr, ptr, ws, None)
    assert step(ptr=None) == capi.EINVAL and "null" in capi.last_error()
    assert step(o=None) == capi.EINVAL
    assert step(mode=3) == capi.EINVAL and "mode" in capi.last_error()
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert step(pw=bad) == capi.EINVAL and "pos_weight" in capi.last_error()
    assert step(ws=need - 1) == capi.ESTATE and "workspace" in capi.last_error()


def test_training_calls_check_arguments_before_the_device():
    """cfg->device is made current only once every other argument has passed: a device that does not exist is not
    what a bad argument reports"""
    lib = capi.load_library()
    cfg = capi.make_config(tskd_b200.ARCH_PRESETS["mycnn5"], device=1000)
    opt = capi.Adam(1e-5, 0.9, 0.999, 1e-8)
    p = ctypes.c_void_p(1)
    assert _fwd(lib, ctypes.byref(cfg), mode=7) == capi.EINVAL and "mode" in capi.last_error()
    assert _bwd(lib, ctypes.byref(cfg), ptr=0) == capi.EINVAL and "null" in capi.last_error()
    rc = lib.b2cnn_train_step_weighted(ctypes.byref(cfg), p, p, p, p, 1, ctypes.byref(opt), 1, p, 4, p, p, 0.0, capi.MODE_SEQUENCE,
                                       None, None, p, p, 1 << 30, None)
    assert rc == capi.EINVAL and "pos_weight" in capi.last_error()


def test_trainable_model_contract_without_a_gpu():
    plain = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"])
    m = tskd_b200.B200TrainableMyCNN(tskd_b200.ARCH_PRESETS["mycnn5"])
    m.load_state_dict(plain.state_dict())
    assert list(m.state_dict().keys()) == list(plain.state_dict().keys())
    assert sum(p.numel() for p in m.parameters() if p.requires_grad) == 5957      # explore_torch.ipynb:2117
    assert m.training is False
    assert m.train() is m and m.training and m.conv1.training
    assert m.eval() is m and not m.training
    with pytest.raises(NotImplementedError):                                      # the inference model stays inference-only
        plain.train()
    with pytest.raises(NotImplementedError):
        tskd_b200.B200TrainableMyCNN(ArchConfig(act="relu"))
    with pytest.raises(NotImplementedError):
        tskd_b200.B200TrainableMyCNN(ArchConfig(affine=True))
    old = tskd_b200.B200TrainableMyCNN(tskd_b200.ARCH_PRESETS["mycnn3"], has_out12=False)
    assert sum(p.numel() for p in old.parameters() if p.requires_grad) == sum(v.numel() for v in old.state_dict().values())


def test_trainable_forward_has_no_cpu_fallback():
    m = tskd_b200.B200TrainableMyCNN(tskd_b200.ARCH_PRESETS["mycnn5"]).train()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 10, 120), torch.full((2,), 50.0))
    named = dict(m.named_parameters())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        tskd_b200.mycnn_train_forward(torch.zeros(2, 10, 120), torch.full((2,), 50.0), [named[k] for k in BLOB_KEYS], m.arch)
    with pytest.raises(ValueError, match="mode"):
        tskd_b200.mycnn_train_forward(torch.zeros(2, 10, 120), torch.full((2,), 50.0), [named[k] for k in BLOB_KEYS], m.arch,
                                      mode="rows")
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m.eval()(torch.zeros(2, 10, 120), torch.full((2,), 50.0))


def test_trainer_pos_weight_is_validated():
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"])
    for bad in (0.0, -2.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="pos_weight"):
            B200Trainer(m, pos_weight=bad)
    with pytest.raises((TypeError, ValueError)):
        B200Trainer(m, pos_weight="heavy")
