"""GPU: b2cnn_slide_push refuses a row pitch of 2^31 samples or more on the tensor-core path, as on the generic path,
before it launches anything."""
import ctypes
from dataclasses import replace

import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_tensorcore_push_rejects_pitch_2_31():
    # W % 4 == 0: phase 0, and a 16-byte aligned segment with an 8-sample pitch would be read in place (not staged);
    # S = 1876 gives more than 32 new features per push, so the tensor-core front end would run on that pitch
    W, S, P, C = 7504, 1876, 4, 3
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    m = tskd_b200.B200MyCNN(replace(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), age_coef=oarch.age_coef),
                            has_out12=oarch.has_out12).to(DEV)
    m.load_state_dict(O.make_ref(oarch, seed=0).state_dict())
    lib, h = m._ensure_handle()
    s = ctypes.c_void_p()
    assert lib.b2cnn_slide_create_path(h, P, S, capi.DTYPE_BF16, capi.PATH_TENSORCORE, ctypes.byref(s)) == capi.OK
    try:
        assert lib.b2cnn_slide_path(s) == capi.PATH_TENSORCORE
        seg = torch.zeros(P, C, S, dtype=torch.bfloat16, device=DEV)     # small: the check comes before any launch
        assert seg.data_ptr() % 16 == 0
        age = torch.full((P,), 50.0, device=DEV)
        out = torch.empty(P, device=DEV)
        em, widx = ctypes.c_int32(0), ctypes.c_int64(-1)
        st = torch.cuda.current_stream().cuda_stream
        rc = lib.b2cnn_slide_push(s, seg.data_ptr(), 1 << 31, age.data_ptr(), P, 0, out.data_ptr(), ctypes.byref(em),
                                  ctypes.byref(widx), st)
        assert rc == capi.EINVAL
        assert em.value == 0
        torch.cuda.synchronize()
    finally:
        lib.b2cnn_slide_destroy(s)
