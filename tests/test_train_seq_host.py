"""CPU: the seq_lengths calls (many sequences in one batch) without a GPU -- the Python validation, the bound _seq
symbols and their refusals before any CUDA call, and the oracle helper against a per-sequence loop of the reference
module."""
import copy
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

import tskd_b200
from tskd_b200 import capi
from oracle import mycnn_torch as O
from oracle.mycnn_c import BLOB_KEYS
from oracle.train_ref import MaskDropout, train_reference
from oracle.train_seq_ref import train_reference_seq


@pytest.mark.parametrize("lens,B,msg", [
    ([3, 4], 8, "add up to 7"),
    ([3, 0, 5], 8, r"seq_lengths\[1\] = 0"),
    ([9, -1], 8, r"seq_lengths\[1\] = -1"),
    ([4.0, 4], 8, r"seq_lengths\[0\] must be an integer, got float"),
    ([True, 7], 8, "got bool"),
    ([], 8, "at least one sequence"),
    ((), 8, "at least one sequence"),
    (torch.tensor([4.0, 4.0]), 8, "integer tensor"),
    (torch.tensor([[4, 4]]), 8, "1-d integer tensor"),
    (torch.tensor([True, False]), 2, "integer tensor"),
    ("44", 8, "list, tuple or integer tensor"),
    (8, 8, "list, tuple or integer tensor"),
])
def test_bad_lengths_are_refused_with_a_clear_message(lens, B, msg):
    with pytest.raises(ValueError, match=msg):
        capi.seq_lengths_array(lens, B)


@pytest.mark.parametrize("lens", [[1, 7, 32, 3, 1, 20], (64,), torch.tensor([10, 54]), torch.tensor([1] * 64, dtype=torch.int32),
                                  [np.int64(60), 4]])
def test_good_lengths_become_a_host_int64_array(lens):
    a = capi.seq_lengths_array(lens, 64)
    assert isinstance(a, ctypes.Array) and a._type_ is ctypes.c_int64
    assert list(a) == [int(v) for v in lens]


def test_seq_symbols_are_bound_and_declared():
    lib = capi.load_library()
    for name in ("b2cnn_train_workspace_bytes_seq", "b2cnn_train_step_seq", "b2cnn_train_forward_seq", "b2cnn_train_backward_seq",
                 "b2cnn_workspace_bytes_seq", "b2cnn_forward_seq"):
        assert name in capi.SYMBOLS
        assert getattr(lib, name).restype is not None


def _cfg():
    return capi.make_config(tskd_b200.ARCH_PRESETS["mycnn5"])


def _arr(v):
    return (ctypes.c_int64 * len(v))(*v)


def test_train_workspace_query_takes_the_lengths():
    lib, cfg = capi.load_library(), _cfg()
    plain = lib.b2cnn_train_workspace_bytes(ctypes.byref(cfg), 64)
    one = lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), 64, _arr([64]), 1)
    many = lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), 64, _arr([1] * 64), 64)
    assert 0 < plain < one <= many                              # the offsets region, then the scan CTAs' rows
    for lens, n in (([32, 31], 2), ([0, 64], 2), ([-1, 65], 2), ([64], 0), ([65], 1)):
        assert lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), 64, _arr(lens), n) == -1
    assert lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), 64, None, 1) == -1
    assert lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), 64, _arr([2 ** 62, 2 ** 62, 64]), 3) == -1    # no overflow


def test_train_calls_refuse_bad_lengths_before_any_cuda_call():
    # fake, never dereferenced device pointers: an EINVAL here proves the lengths are checked before the first CUDA call
    lib, cfg = capi.load_library(), _cfg()
    p = ctypes.c_void_p(16)
    opt = capi.Adam(1e-3, 0.9, 0.999, 1e-8)
    for lens, n in (([3, 4], 2), ([8, 0], 2), ([8], 0), (None, 1)):
        arr = None if lens is None else _arr(lens)
        rc = lib.b2cnn_train_step_seq(ctypes.byref(cfg), p, p, p, p, 1, ctypes.byref(opt), 1, p, 8, p, p, None, arr, n, None, None, p, p,
                                      1 << 30, None)
        assert rc == capi.EINVAL, (lens, capi.last_error())
        assert "seq_lengths" in capi.last_error()
        assert lib.b2cnn_train_forward_seq(ctypes.byref(cfg), p, p, 8, p, arr, n, None, None, p, p, 1 << 30, None) == capi.EINVAL
        assert lib.b2cnn_train_backward_seq(ctypes.byref(cfg), p, p, 8, p, arr, n, None, None, p, p, None, None, 0, p, 1 << 30,
                                            None) == capi.EINVAL
    # a workspace sized by the query without lengths is too small for the _seq call: B2CNN_ESTATE, still before CUDA
    need = lib.b2cnn_train_workspace_bytes(ctypes.byref(cfg), 8)
    rc = lib.b2cnn_train_forward_seq(ctypes.byref(cfg), p, p, 8, p, _arr([5, 3]), 2, None, None, p, p, need, None)
    assert rc == capi.ESTATE and "b2cnn_train_workspace_bytes_seq" in capi.last_error()
    # a bad pos_weight is refused like b2cnn_train_step_weighted's
    bad = ctypes.c_float(-1.0)
    need = lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), 8, _arr([5, 3]), 2)
    rc = lib.b2cnn_train_step_seq(ctypes.byref(cfg), p, p, p, p, 1, ctypes.byref(opt), 1, p, 8, p, p, ctypes.byref(bad), _arr([5, 3]), 2,
                                  None, None, p, p, need, None)
    assert rc == capi.EINVAL and "pos_weight" in capi.last_error()


def test_python_refuses_seq_lengths_in_independent_mode_without_a_gpu():
    arch = tskd_b200.ARCH_PRESETS["mycnn5"]
    x, age = torch.zeros(4, 10, 120), torch.zeros(4)
    params = [torch.zeros(s) for s in arch.param_shapes().values()][:len(BLOB_KEYS)]
    with pytest.raises(ValueError, match="mode='sequence'"):
        tskd_b200.mycnn_train_forward(x, age, params, arch, "independent", seq_lengths=[2, 2])
    m = tskd_b200.B200MyCNN(arch)
    with pytest.raises(ValueError, match="mode='sequence'"):
        m.predict(x, age, mode="independent", seq_lengths=[4])
    m.batch_mode = "independent"
    with pytest.raises(ValueError, match="batch_mode"):
        m(x, age, seq_lengths=[4])
    t = tskd_b200.B200TrainableMyCNN(arch)
    t.batch_mode = "independent"
    t.train()
    with pytest.raises(ValueError, match="batch_mode"):
        t(x, age, seq_lengths=[4])


def _ref(kind, C, W, seed=0):
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    ref.dropout = MaskDropout()
    ref.train()
    return ref


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_oracle_helper_is_a_per_sequence_loop_of_the_reference(dtype):
    ref = _ref("mycnn5", 10, 120)
    a = O.stretched(O.ARCHS["mycnn5"], 10, 120)
    lens = [1, 7, 3, 1, 5]
    B = sum(lens)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, 10, 120, generator=g)
    age = torch.rand(B, generator=g) * 60 + 20
    y = (torch.rand(B, generator=g) > 0.5).float()
    m1 = torch.bernoulli(torch.full((B, 4, a.p1), 0.9), generator=g) / 0.9
    m2 = torch.bernoulli(torch.full((B, a.l_out), 0.9), generator=g) / 0.9
    got = train_reference_seq(ref, x, age, lens, m1, m2, target=y, pos_weight=13.5, dtype=dtype)
    # the same thing by hand: the reference module itself, once per sequence, the losses summed and divided by B
    m = copy.deepcopy(ref).to(dtype)
    xd, ad = x.to(dtype).requires_grad_(), age.to(dtype).requires_grad_()
    zs, o = [], 0
    for n in lens:
        m.dropout.set(m1[o:o + n].to(dtype), m2[o:o + n].to(dtype))
        zs.append(m(xd[o:o + n], ad[o:o + n]).reshape(-1))
        o += n
    z = torch.cat(zs)
    assert torch.equal(got["z"], z.detach())
    loss = nn.BCEWithLogitsLoss(pos_weight=torch.tensor(13.5, dtype=dtype))(z, y.to(dtype))
    loss.backward()
    assert torch.equal(got["bce_pw"]["loss"], loss.detach())
    named = dict(m.named_parameters())
    for k in BLOB_KEYS:
        torch.testing.assert_close(got["bce_pw"]["grads"][k], named[k].grad, rtol=0, atol=0)
    torch.testing.assert_close(got["bce_pw"]["dx"], xd.grad, rtol=0, atol=0)
    torch.testing.assert_close(got["bce_pw"]["dage"], ad.grad, rtol=0, atol=0)


def test_oracle_helper_special_cases():
    ref = _ref("mycnn2", 7, 120)
    g = torch.Generator().manual_seed(5)
    x, age = torch.randn(6, 7, 120, generator=g), torch.rand(6, generator=g) * 60 + 20
    r = torch.randn(6, generator=g)
    whole = train_reference(ref, x, age, "sequence", dz=r)
    one = train_reference_seq(ref, x, age, [6], dz=r)
    assert torch.equal(whole["z"], one["z"])
    indep = train_reference(ref, x, age, "independent", dz=r)
    ones = train_reference_seq(ref, x, age, [1] * 6, dz=r)
    assert torch.equal(indep["z"], ones["z"])
    for k in BLOB_KEYS:
        torch.testing.assert_close(ones["dz"]["grads"][k], indep["dz"]["grads"][k], rtol=1e-12, atol=1e-15)
    with pytest.raises(ValueError):
        train_reference_seq(ref, x, age, [2, 3], dz=r)
