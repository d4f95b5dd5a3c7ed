"""GPU: which kernels a forward call runs (DESIGN.md §2, the router in csrc/b2cnn_api.cu) and the workspace it may
touch.  Every row of the route table is called through the raw C ABI with a workspace of exactly the queried size
followed by a guard tail, so a route that writes past its own layout fails here instead of corrupting memory it does
not own.  The tail is larger than any staging copy the library can make, so even such a write stays inside the
test's own allocation."""
from dataclasses import replace

import pytest
import torch

import tskd_b200
from tskd_b200 import capi
from oracle import mycnn_torch as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
IND, SEQ = capi.MODE_INDEPENDENT, capi.MODE_SEQUENCE
GUARD = 0xA5

_models = {}


def _model(kind, C, W):
    key = (kind, C, W)
    if key not in _models:
        oarch = O.stretched(O.ARCHS[kind], C, W)
        arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
        m = tskd_b200.B200MyCNN(arch, has_out12=oarch.has_out12).to(DEV)
        m.load_state_dict(O.make_ref(oarch, seed=5).state_dict())
        _models[key] = m
    return _models[key]


def _configure(m, path="auto", **opts):
    m.set_path(path)
    for k, v in {"tc_fused": 1, "small_kernel": 1, **opts}.items():
        m.set_option(k, v)


def _windows(B, C, W, dtype, pitch=None):
    """[B, C, W] windows, contiguous or a view of a [B, C, pitch] buffer (the pad holds NaN: it must never be read)."""
    x = tskd_b200.synth.make_windows(B, C, W, "physio", seed=B + W, dtype=dtype, device=DEV)
    if pitch is None or pitch == W:
        return x
    buf = torch.full((B, C, pitch), float("nan"), dtype=dtype, device=DEV)
    xp = buf.as_strided((B, C, W), (C * pitch, pitch, 1))
    xp.copy_(x)
    return xp


def _call(m, x, mode, need):
    """One b2cnn_forward_pitched call with `need` bytes of workspace followed by a guard tail.  Returns
    (rc, out, tail_intact)."""
    lib, h = m._ensure_handle()
    B, C, W = x.shape
    pitch = x.stride(1)
    tail = B * C * ((W + 7) // 8 * 8) * 2 + 4096                 # more than any staging copy of these windows
    ws = torch.full((need + tail,), GUARD, dtype=torch.uint8, device=DEV)
    out = torch.full((B,), 12345.0, device=DEV)
    age = tskd_b200.synth.make_ages(B, seed=B, device=DEV)
    dtype = capi.DTYPE_BF16 if x.dtype == BF else capi.DTYPE_F32
    rc = lib.b2cnn_forward_pitched(h, x.data_ptr(), dtype, B, pitch, age.data_ptr(), B, mode, 0, out.data_ptr(),
                                   ws.data_ptr(), need, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, out, bool((ws[need:] == GUARD).all())


def _need_for(m, B, mode, dtype):
    lib, h = m._ensure_handle()
    return int(lib.b2cnn_workspace_bytes_for(h, B, mode, capi.DTYPE_BF16 if dtype == BF else capi.DTYPE_F32))


def _need_any(m, B, mode):
    lib, h = m._ensure_handle()
    return int(lib.b2cnn_workspace_bytes(h, B, mode))


# (kind, C, W, dtype, B, mode, path, options, row pitch or None) -> (last_path, launches); EARCH: refused.
# Launches: batch / small 1; generic front end 1 + projection, reduction, LSTM head 3; streaming kernels (fp32 stream,
# bf16 fused) 1 + exact recompute of flagged windows 1 + head 1 (a sequence scan reduces the ranges first: + 1);
# unfused tensor-core front end 1 + flag compaction 1 + exact recompute 1 + the generic head 3; + 1 staging copy for
# bf16 rows whose pitch is not a multiple of 8 samples.
ROUTES = [
    # short windows: the batch kernel takes B >= 8 independent windows before the small kernel is considered
    ("mycnn5", 10, 120, F32, 8, IND, "auto", {}, None, ("generic", 1)),
    ("mycnn5", 10, 120, F32, 256, IND, "auto", {}, None, ("generic", 1)),
    ("mycnn5", 10, 120, BF, 4, IND, "auto", {}, None, ("generic", 1)),            # small
    ("mycnn5", 10, 120, F32, 1, SEQ, "auto", {}, None, ("generic", 1)),           # small: a one-window sequence
    ("mycnn5", 10, 120, F32, 8, SEQ, "auto", {}, None, ("generic", 4)),           # neither: generic front end + head
    ("mycnn5", 10, 120, F32, 8, IND, "auto", {"small_kernel": 0}, None, ("generic", 4)),
    ("mycnn5", 10, 120, F32, 8, IND, "generic", {}, None, ("generic", 1)),        # path=generic keeps the short kernels
    # a short window the tensor cores could take: small under auto, skipped under path=tensorcore
    ("mycnn5", 3, 1528, BF, 5, IND, "auto", {}, None, ("generic", 1)),
    ("mycnn5", 3, 1528, BF, 5, IND, "tensorcore", {}, None, ("tensorcore", 3)),
    ("mycnn5", 3, 1528, BF, 300, IND, "auto", {}, None, ("tensorcore", 3)),
    # bf16: fused, unfused, staging
    ("mycnn5", 3, 7504, BF, 64, IND, "auto", {}, None, ("tensorcore", 3)),
    ("mycnn5", 3, 7504, BF, 64, SEQ, "auto", {}, None, ("tensorcore", 4)),
    ("mycnn5", 3, 7504, BF, 64, IND, "generic", {}, None, ("generic", 4)),
    ("mycnn5", 3, 7500, BF, 64, IND, "auto", {}, None, ("tensorcore", 4)),        # W % 8 == 4: staged
    ("mycnn5", 3, 7500, BF, 64, IND, "auto", {}, 7504, ("tensorcore", 3)),        # padded rows: not staged
    ("mycnn5", 3, 7500, BF, 64, SEQ, "auto", {}, None, ("tensorcore", 5)),
    ("mycnn5", 3, 7500, BF, 64, IND, "auto", {"tc_fused": 0}, None, ("tensorcore", 7)),
    ("mycnn5", 3, 7504, BF, 64, IND, "tensorcore", {"tc_fused": 0}, None, ("tensorcore", 6)),
    ("mycnn5", 4, 3000, BF, 64, IND, "auto", {}, None, ("tensorcore", 6)),        # C = 4: unfused only
    ("mycnn5", 4, 3000, BF, 64, SEQ, "auto", {}, None, ("tensorcore", 6)),
    ("mycnn5", 4, 3000, F32, 64, IND, "auto", {}, None, ("generic", 4)),          # ... and no fp32 stream kernel
    ("mycnn5", 4, 3000, F32, 64, IND, "tensorcore", {}, None, "EARCH"),
    # MyCNN2/3/4 geometry has no unfused tensor-core kernel
    ("mycnn3", 3, 7504, BF, 64, IND, "auto", {}, None, ("tensorcore", 3)),
    ("mycnn3", 3, 7504, BF, 64, IND, "auto", {"tc_fused": 0}, None, ("generic", 4)),
    ("mycnn3", 3, 7504, BF, 64, IND, "tensorcore", {"tc_fused": 0}, None, "EARCH"),
    ("mycnn3", 3, 7504, F32, 64, SEQ, "auto", {"tc_fused": 0}, None, ("stream", 4)),   # tc_fused is a bf16 option
    # fp32: the stream kernel needs rows that are a multiple of 16 bytes
    ("mycnn5", 3, 7504, F32, 64, IND, "auto", {}, None, ("stream", 3)),
    ("mycnn5", 3, 7504, F32, 64, SEQ, "auto", {}, None, ("stream", 4)),
    ("mycnn5", 3, 7504, F32, 64, IND, "tensorcore", {}, None, ("stream", 3)),
    ("mycnn5", 3, 7502, F32, 64, IND, "auto", {}, None, ("generic", 4)),
    ("mycnn5", 3, 7502, F32, 64, IND, "auto", {}, 7504, ("stream", 3)),
    ("mycnn5", 3, 7502, F32, 64, IND, "tensorcore", {}, None, "EARCH"),
]


def _route_id(r):
    kind, C, W, dtype, B, mode, path, opts, pitch, _ = r
    o = ",".join(f"{k}={v}" for k, v in opts.items())
    return (f"{kind}-C{C}-W{W}-{'bf16' if dtype == BF else 'f32'}-B{B}-{'seq' if mode else 'ind'}-{path}"
            + (f"-{o}" if o else "") + (f"-pitch{pitch}" if pitch else ""))


@pytest.mark.parametrize("kind,C,W,dtype,B,mode,path,opts,pitch,want", ROUTES, ids=[_route_id(r) for r in ROUTES])
def test_route_table_and_exact_workspace(kind, C, W, dtype, B, mode, path, opts, pitch, want):
    """Each route runs with a workspace of exactly b2cnn_workspace_bytes_for() bytes, writes nothing past it, reports
    the expected last_path and launch count, and computes what predict() computes."""
    m = _model(kind, C, W)
    _configure(m, path, **opts)
    x = _windows(B, C, W, dtype, pitch)
    need = _need_for(m, B, mode, dtype)
    assert need > 0
    rc, out, tail_ok = _call(m, x, mode, need)
    assert tail_ok, "the call wrote past the queried workspace size"
    if want == "EARCH":
        assert rc == capi.EARCH
        assert bool((out == 12345.0).all())
        return
    assert rc == capi.OK, capi.load_library().b2cnn_last_error()
    assert (m.last_path, m.gpu_launches) == want
    ref = m.predict(x, tskd_b200.synth.make_ages(B, seed=B, device=DEV), mode="sequence" if mode else "independent")
    assert m.last_path == want[0]
    assert torch.equal(out, ref)


def test_misaligned_bf16_pitch_needs_the_dtype_blind_workspace():
    """bf16 rows 7508 samples apart (not a multiple of 8) are staged into aligned rows.  The staging region is not part
    of the exact size for contiguous W = 7504 windows: such a call is refused with that size and runs with the
    dtype-blind one, bit for bit like the contiguous call."""
    B, C, W, P = 64, 3, 7504, 7508
    m = _model("mycnn5", C, W)
    _configure(m)
    x = _windows(B, C, W, BF, P)
    rc, out, tail_ok = _call(m, x, IND, _need_for(m, B, IND, BF))
    assert rc == capi.ESTATE and tail_ok and bool((out == 12345.0).all())
    assert b"b2cnn_workspace_bytes()" in capi.load_library().b2cnn_last_error()
    xc = x.contiguous()
    rc, want, _ = _call(m, xc, IND, _need_for(m, B, IND, BF))
    assert rc == capi.OK and m.last_path == "tensorcore"
    launches_c = m.gpu_launches
    rc, out, tail_ok = _call(m, x, IND, _need_any(m, B, IND))
    assert rc == capi.OK and tail_ok
    assert m.last_path == "tensorcore" and m.gpu_launches == launches_c + 1         # + the staging copy
    assert torch.equal(out, want)


def test_misaligned_f32_pitch_needs_the_dtype_blind_workspace():
    """fp32 rows 7506 samples apart cannot be described by a TMA map: the call takes the generic kernels, whose feature
    rows the exact size for contiguous windows (stream kernel) does not hold."""
    B, C, W, P = 64, 3, 7504, 7506
    m = _model("mycnn5", C, W)
    _configure(m)
    x = _windows(B, C, W, F32, P)
    rc, out, tail_ok = _call(m, x, IND, _need_for(m, B, IND, F32))
    assert rc == capi.ESTATE and tail_ok and bool((out == 12345.0).all())
    rc, out, tail_ok = _call(m, x, IND, _need_any(m, B, IND))
    assert rc == capi.OK and tail_ok and m.last_path == "generic"
    _configure(m, "generic")
    rc, want, _ = _call(m, x.contiguous(), IND, _need_for(m, B, IND, F32))
    _configure(m)
    assert rc == capi.OK and m.last_path == "generic"
    assert torch.equal(out, want)


def test_dtype_blind_size_covers_every_exact_size():
    for kind, C, W in [("mycnn5", 3, 7504), ("mycnn5", 3, 7500), ("mycnn5", 4, 3000), ("mycnn3", 3, 7504), ("mycnn5", 10, 120)]:
        m = _model(kind, C, W)
        _configure(m)
        for B in (1, 64, 4096):
            for mode in (IND, SEQ):
                blind = _need_any(m, B, mode)
                assert blind >= max(_need_for(m, B, mode, BF), _need_for(m, B, mode, F32))
                if C <= 4:                                    # tensor-core state prepared: the staging rows are counted
                    assert blind >= B * C * ((W + 7) // 8 * 8) * 2


def test_features_rejects_a_bad_dtype():
    m = _model("mycnn5", 3, 7504)
    _configure(m)
    lib, h = m._ensure_handle()
    x = _windows(4, 3, 7504, BF)
    feats = torch.zeros(4, m.arch.l_out, device=DEV)
    assert lib.b2cnn_features(h, x.data_ptr(), 2, 4, feats.data_ptr(), None) == capi.EINVAL
    assert lib.b2cnn_features(h, x.data_ptr(), capi.DTYPE_BF16, 4, feats.data_ptr(), None) == capi.OK
    torch.cuda.synchronize()
    assert m.last_path == "tensorcore"


def test_stream_f32_option_is_gone():
    m = _model("mycnn5", 3, 7504)
    lib, h = m._ensure_handle()
    assert lib.b2cnn_set_option(h, b"stream_f32", 0) == capi.EINVAL
