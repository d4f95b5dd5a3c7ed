"""GPU: the exact CUDA-core inference kernels element by element against the float64 reference of oracle/infer_ref.py,
across everything the C ABI accepts beyond the reference's own layer stack: the three activations (tanh, relu,
identity), the folded eval-BatchNorm (B2CNN_FLAG_AFFINE, always with a negative scale: pooling before it would pick the
minimum), and conv/pool geometries off the reference's two.

The kernels (DESIGN.md §2 and §5):
  * the templated generic front end ``frontend_kernel`` (csrc/b2cnn_generic.cu): RUN = 1 below 96 final positions and
    RUN = 4 from 96 on, a fixed C or the CT = 0 instantiation, the pooled-first branch and the affine branch, window
    tiles of 508 final positions;
  * the runtime-geometry generic front end ``frontend_any_kernel``: any pool (1,1), (2,3), (4,3), (2,1), C = 16;
  * the single-launch ``small`` kernel (csrc/b2cnn_small.cu) up to each of its bounds, and one step past each;
  * the one-warp-per-window ``batch`` kernel (csrc/b2cnn_batch.cu): its six (C, k1, pool_k) instantiations, vector and
    scalar loads, pitched rows, the grid-stride loop.

Every comparison is tests/test_gpu_infer_elem.py's (oracle/train_ref.py::check_elems): |got - truth| <=
8 |ref32 - truth| + beta max|truth| per element, beta = 2^-20, NaN and infinities exactly where the float64 truth has
them; the smallest passing beta and the number of finite elements judged are printed (pytest -s).  Batch-as-sequence
is judged on windows whose NaN / inf samples sit in the last window only, so the scan stays finite up to the last step
(a NaN in window 0 would make every logit of the scan NaN).  Every test asserts its route: last_path and the launch count (1 for small / batch, 4 for the generic
front end + projection, reduction and LSTM head, 1 for features()).  A case never depends on the tensor-core kernels:
the front-end cases run under path=generic with small_kernel=0, the others take no tensor-core route (relu, identity,
affine or a geometry the tensor-core kernels lack)."""
from collections import namedtuple

import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import centre_affine, infer_reference, random_affine
from oracle.train_ref import BETA, check_elems
from tskd_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32
COEF = 1e-4                                                      # age_coef of every case

# ------------------------------------------------------------------ cases
# geo: (C, k1, k2, pool_k, pool_s, W); route: "front" = the generic front end + head (path=generic, small_kernel=0),
# "short" = the small or batch kernel (one launch; which one is DESIGN.md §2: batch for B >= 8 on its geometries),
# "general" = auto routing that must fall through to the generic front end + head (a short kernel's bound exceeded);
# bad: NaN at the first / last sample, +inf, -inf; age: "rand", "kink" (age * coef + 1 == 0 and < 0), "nan";
# pitch: 0 for contiguous rows, else the row pitch in elements of a NaN-padded buffer (the pad must never be read)
Case = namedtuple("Case", "route geo dtype B act aff seed bad age pitch", defaults=(False, "rand", 0))
M5, M3 = (10, 5, 3, 2), (5, 5, 2, 2)                             # (k1, k2, pool_k, pool_s) of MyCNN5 and MyCNN2/3/4
G = lambda C, kk, W: (C,) + kk + (W,)                            # noqa: E731

CASES = {
    # ---- templated frontend_kernel: CT = 10 / 3 / 7 and CT = 0, RUN = 1 / 4, one and several 508-position tiles
    "t-m5-c10-w120-f32-tanh": Case("front", G(10, M5, 120), F32, 8, "tanh", False, 1, True, "kink"),
    "t-m5-c10-w120-bf16-relu-aff": Case("front", G(10, M5, 120), BF, 5, "relu", True, 2, True),
    "t-m5-c3-w400-f32-identity-aff": Case("front", G(3, M5, 400), F32, 4, "identity", True, 3, True),     # L = 95: RUN = 1
    "t-m5-c3-w404-bf16-relu": Case("front", G(3, M5, 404), BF, 4, "relu", False, 4, True),               # L = 96: RUN = 4
    "t-m5-c3-w404-f32-tanh-aff": Case("front", G(3, M5, 404), F32, 4, "tanh", True, 5, age="nan"),
    "t-m5-c3-w2056-bf16-identity-aff": Case("front", G(3, M5, 2056), BF, 3, "identity", True, 6, True),  # L = 509
    "t-m5-c3-w2056-f32-tanh": Case("front", G(3, M5, 2056), F32, 3, "tanh", False, 7, True),
    "t-m5-c3-w4084-bf16-relu-aff-pitched": Case("front", G(3, M5, 4084), BF, 3, "relu", True, 8, True, pitch=4088),  # L = 1016
    "t-m5-c3-w4084-f32-identity": Case("front", G(3, M5, 4084), F32, 3, "identity", False, 9, True),
    "t-m5-c5-w800-bf16-tanh-aff": Case("front", G(5, M5, 800), BF, 4, "tanh", True, 10, True),          # CT = 0
    "t-m3-c7-w700-f32-relu": Case("front", G(7, M3, 700), F32, 4, "relu", False, 11, True),
    "t-m3-c5-w1000-f32-relu-aff": Case("front", G(5, M3, 1000), F32, 4, "relu", True, 12, True),         # CT = 0
    "t-m3-c2-w1533-bf16-identity": Case("front", G(2, M3, 1533), BF, 5, "identity", False, 13, True),    # CT = 0
    "t-m3-c2-w300-f32-tanh-aff": Case("front", G(2, M3, 300), F32, 8, "tanh", True, 14, True, "kink"),   # CT = 0, RUN = 1
    # ---- frontend_any_kernel
    "a-p11-w600-f32-relu": Case("front", (2, 4, 3, 1, 1, 600), F32, 3, "relu", False, 21, True),         # L = 595: 2 tiles
    "a-p11-w600-bf16-identity-aff": Case("front", (2, 4, 3, 1, 1, 600), BF, 3, "identity", True, 22, True),
    "a-p23-w60-f32-tanh-aff": Case("front", (3, 4, 3, 2, 3, 60), F32, 8, "tanh", True, 23, True, "kink"),
    "a-p23-w5000-bf16-relu": Case("front", (3, 4, 3, 2, 3, 5000), BF, 3, "relu", False, 25, True),       # L = 555: 2 tiles
    "a-p23-w5000-f32-identity-aff": Case("front", (3, 4, 3, 2, 3, 5000), F32, 3, "identity", True, 25, True),
    "a-p43-w700-f32-identity": Case("front", (4, 6, 4, 4, 3, 700), F32, 4, "identity", False, 26, True),
    "a-p43-w700-bf16-tanh-aff": Case("front", (4, 6, 4, 4, 3, 700), BF, 4, "tanh", True, 27, True, "nan"),
    "a-p21-w300-bf16-relu-aff": Case("front", (3, 7, 2, 2, 1, 300), BF, 4, "relu", True, 28, True),
    "a-p21-w301-f32-tanh-pitched": Case("front", (3, 7, 2, 2, 1, 301), F32, 4, "tanh", False, 29, True, pitch=304),
    "a-c16-w900-f32-relu-aff": Case("front", (16, 3, 8, 3, 2, 900), F32, 3, "relu", True, 30, True),
    "a-c16-w900-bf16-identity": Case("front", (16, 3, 8, 3, 2, 900), BF, 3, "identity", False, 31, True),
    # ---- small: each activation with and without affine, pitched rows, B = 1, the bounds and one step past each
    "s-tanh": Case("short", (4, 6, 4, 3, 3, 500), F32, 7, "tanh", False, 41, True, "kink"),
    "s-tanh-aff": Case("short", (4, 6, 4, 3, 3, 500), BF, 5, "tanh", True, 42),
    "s-relu": Case("short", (4, 6, 4, 3, 3, 500), BF, 5, "relu", False, 43, True),
    "s-relu-aff": Case("short", (4, 6, 4, 3, 3, 500), F32, 5, "relu", True, 44, age="nan"),
    "s-identity": Case("short", (4, 6, 4, 3, 3, 500), F32, 5, "identity", False, 45, True),
    "s-identity-aff": Case("short", (4, 6, 4, 3, 3, 500), BF, 5, "identity", True, 46, True),
    "s-relu-aff-pitched": Case("short", (4, 6, 4, 3, 3, 501), F32, 4, "relu", True, 47, True, pitch=504),
    "s-b1-identity-aff": Case("short", (3, 5, 3, 2, 2, 900), F32, 1, "identity", True, 48),
    "s-b256": Case("short", (2, 5, 3, 2, 2, 700), F32, 256, "relu", False, 49, True),
    "g-b257": Case("general", (2, 5, 3, 2, 2, 700), F32, 257, "relu", False, 49, True),
    "s-cw8192": Case("short", (4, 3, 3, 2, 2, 2048), BF, 3, "identity", True, 50, True),
    "g-cw8196": Case("general", (4, 3, 3, 2, 2, 2049), BF, 3, "identity", True, 50, True),
    "s-smem96k": Case("short", (1, 3, 3, 2, 2, 7537), F32, 3, "tanh", True, 51, True),     # 98300 of 98304 bytes
    "g-smem96k": Case("general", (1, 3, 3, 2, 2, 7538), F32, 3, "tanh", True, 51, True),
    "s-l2048": Case("short", (1, 3, 3, 1, 1, 2052), F32, 3, "relu", True, 52, True),       # L = 2048
    "g-l2049": Case("general", (1, 3, 3, 1, 1, 2053), F32, 3, "relu", True, 52, True),
    # ---- batch: the six instantiations, B = 8 / not a multiple of 8 / many windows per warp, loads, W bounds
    "b-c10-k10-p3-relu": Case("short", G(10, M5, 120), F32, 8, "relu", False, 63, True),
    "b-c10-k5-p2-identity-bf16": Case("short", G(10, M3, 120), BF, 13, "identity", False, 62, True, "kink"),
    "b-c7-k5-p2-relu-w128": Case("short", G(7, M3, 128), F32, 8, "relu", False, 63, True),        # L1 = 124
    "b-c7-k10-p3-identity-w100": Case("short", G(7, M5, 100), F32, 21, "identity", False, 64, True, "nan"),
    "b-c3-k10-p3-relu-bf16-w122": Case("short", G(3, M5, 122), BF, 37, "relu", False, 65, True),  # bf16 W % 8 != 0: scalar
    "b-c3-k5-p2-identity-b12000": Case("short", G(3, M3, 120), F32, 12000, "identity", False, 66, True),
    "b-c10-k10-p3-tanh-pitch128": Case("short", G(10, M5, 120), F32, 9, "tanh", False, 67, True, pitch=128),  # vector, XP != W
    "b-c7-k5-p2-relu-pitched-w118": Case("short", G(7, M3, 118), F32, 11, "relu", False, 68, True, pitch=120),  # scalar
    "b-c3-k5-p2-tanh-bf16-w128": Case("short", G(3, M3, 128), BF, 16, "tanh", False, 69, True),   # bf16 vector loads
    "b-c10-k5-p2-identity-b8": Case("short", G(10, M3, 120), F32, 8, "identity", False, 70),
    # ---- the geometry whose generic tile only fits shared memory for short enough windows (see the refusal test)
    "g-c16-p44-w2430": Case("general", (16, 3, 8, 4, 4, 2430), F32, 3, "relu", True, 71, True),   # L = 150
}
BIG_TILE = (16, 3, 8, 4, 4, 4830)                                 # L = 300: a 508-position tile needs > 220 KB


def _oarch(geo):
    C, k1, k2, pk, ps, W = geo
    return O.RefArch(in_channels=C, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=W, age_coef=COEF, has_out12=False)


def _model(ref, act, aff, path="auto", small=1):
    a = ref.arch
    arch = tskd_b200.ArchConfig(in_channels=a.in_channels, k1=a.k1, k2=a.k2, pool_k=a.pool_k, pool_s=a.pool_s,
                                window=a.window, age_coef=a.age_coef, act=act, affine=aff is not None)
    assert arch.l_out == a.l_out
    m = tskd_b200.B200MyCNN(arch, has_out12=False, path=path).to(DEV)
    sd = dict(ref.state_dict())
    if aff is not None:
        sd.update(zip(("affine1_scale", "affine1_shift", "affine2_scale", "affine2_shift"), aff))
    m.load_state_dict(sd)
    m.set_option("small_kernel", small)
    return m


def _inject(x):
    """NaN at the first sample of the first window and the last sample of the third, +inf mid-window, -inf in the last"""
    B, C, W = x.shape
    x[0, 0, 0] = float("nan")
    x[min(2, B - 1), C - 1, W - 1] = float("nan")
    x[min(3, B - 1), 0, W // 2] = float("inf")
    x[B - 1, C - 1, W // 3] = float("-inf")


def _ages(c):
    g = torch.Generator().manual_seed(c.seed)
    age = torch.rand(c.B, generator=g) * 65 + 15
    if c.age == "kink":                 # age * coef + 1 == 0 (in float64 and float32) in a clean and a bad window, < 0
        age[1] = age[2] = -1.0 / COEF
        age[c.B - 3] = -3.0 / COEF
    elif c.age == "nan":
        age[c.B // 2] = float("nan")
    return age


def _modes(c):
    """batch modes a case is judged in: sequence wherever its route takes it (the short kernels: B = 1 only)"""
    return ["independent"] + (["sequence"] if (c.route != "short" and c.B > 1) or c.B == 1 else [])


def build_case(name):
    """(ref, affine, age, {mode: (x, truth, ref32)}): per batch mode the windows, the float64 truth and the float32
    reference.  A sequence scan carries a NaN to every later step, so the sequence windows hold the bad samples in
    their last window only: the first B - 1 logits judge finite values, the last one the NaN / inf pattern."""
    c = CASES[name]
    ref = O.make_ref(_oarch(c.geo), seed=c.seed)
    clean = tskd_b200.synth.make_windows(c.B, c.geo[0], c.geo[-1], "normal", seed=c.seed)
    aff = centre_affine(ref, clean, c.act, random_affine(c.seed)) if c.aff else None
    x, xs = clean.clone(), clean.clone()
    if c.bad:
        _inject(x)
        _inject(xs[-1:])
    age = _ages(c)
    data = {}
    for md, w in (("independent", x), ("sequence", xs)):
        if md in _modes(c):
            w = w.to(c.dtype)
            data[md] = (w, infer_reference(ref, w, age, md, act=c.act, affine=aff),
                        infer_reference(ref, w, age, md, torch.float32, act=c.act, affine=aff))
    # the case must judge something: finite features, under relu not (almost) all clamped to 0, finite nonzero logits
    f = data["independent"][1]["features"]
    fin = f[torch.isfinite(f)]
    assert fin.numel() >= f.numel() // 2 and (fin != 0).float().mean() >= 0.2, name
    for md, (_, t, _) in data.items():
        z = t["z"]
        assert (z[torch.isfinite(z)] != 0).any(), (name, md)
        if md == "sequence":                               # at most one NaN age among the first B - 1 steps
            assert int(torch.isfinite(z[:-1]).sum()) >= c.B - 2, (name, md)
    return ref, aff, age, data


@pytest.fixture(scope="module")
def case_data():
    """the float64 truth of a case is computed once (one case's windows are kept at a time)"""
    cache = {}

    def get(name):
        if name not in cache:
            cache.clear()
            cache[name] = build_case(name)
        return cache[name]
    yield get
    cache.clear()


def _to_dev(c, x):
    if not c.pitch:
        return x.to(DEV)
    B, C, W = x.shape
    buf = torch.full((B, C, c.pitch), float("nan"), dtype=x.dtype, device=DEV)
    xp = buf[:, :, :W]
    xp.copy_(x)
    assert not xp.is_contiguous()
    return xp


def _route(m):
    return m.last_path, m.gpu_launches


@pytest.mark.parametrize("name", list(CASES))
def test_logits_and_features(case_data, name):
    c = CASES[name]
    ref, aff, age, data = case_data(name)
    x, truth, ref32 = data["independent"]
    front = c.route == "front"
    m = _model(ref, c.act, aff, path="generic" if front else "auto", small=0 if front else 1)
    xd, ad = _to_dev(c, x), age.to(DEV)
    want = ("generic", 1 if c.route == "short" else 4)
    z = m.predict(xd, ad)
    assert _route(m) == want, (name, _route(m), want)
    pairs = [("z", z, truth["z"], ref32["z"], BETA)]
    if c.route == "short":
        p = m.predict(xd, ad, return_prob=True)
        assert _route(m) == want
        pairs.append(("prob", p, torch.sigmoid(truth["z"]), torch.sigmoid(ref32["z"]), BETA))
    f = m.features(xd)
    assert _route(m) == ("generic", 1)
    pairs.append(("features", f, truth["features"], ref32["features"], BETA))
    if "sequence" in data:
        xs, ts, rs = data["sequence"]
        zs = m.predict(_to_dev(c, xs), ad, mode="sequence")
        assert _route(m) == want
        pairs.append(("z sequence", zs, ts["z"], rs["z"], BETA))
    if c.route == "short":                                # the same windows through the generic front end + head
        m.set_option("small_kernel", 0)
        z4 = m.predict(xd, ad)
        assert _route(m) == ("generic", 4)
        pairs.append(("z generic", z4, truth["z"], ref32["z"], BETA))
    print(f"{name}: route {want}, L = {m.arch.l_out}")
    check_elems(pairs, name)


# ------------------------------------------------------------------ refusals
def _raw_forward(m, x, age, out_fill=12345.0):
    """one b2cnn_forward with the dtype-blind workspace size; returns (rc, out, message)"""
    lib, h = m._ensure_handle()
    B = x.shape[0]
    dtype = capi.DTYPE_BF16 if x.dtype == BF else capi.DTYPE_F32
    ws = torch.empty(int(lib.b2cnn_workspace_bytes(h, B, capi.MODE_INDEPENDENT)), dtype=torch.uint8, device=DEV)
    out = torch.full((B,), out_fill, device=DEV)
    rc = lib.b2cnn_forward(h, x.data_ptr(), dtype, B, age.data_ptr(), age.numel(), capi.MODE_INDEPENDENT, 0,
                           out.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, out, capi.last_error()


@pytest.mark.parametrize("act,affine", [("relu", False), ("identity", False), ("tanh", True)])
def test_tensorcore_path_refuses_other_activations_and_affine(act, affine):
    """the tensor-core kernels exist for tanh without affine only: path=tensorcore is B2CNN_EARCH, out untouched"""
    geo = G(3, M5, 7504)
    ref = O.make_ref(_oarch(geo), seed=80)
    x = tskd_b200.synth.make_windows(4, 3, 7504, "normal", seed=80, dtype=BF, device=DEV)
    aff = random_affine(80) if affine else None
    m = _model(ref, act, aff, path="tensorcore")
    rc, out, msg = _raw_forward(m, x, torch.full((1,), 65.0, device=DEV))
    assert rc == capi.EARCH and "tensor-core" in msg, (rc, msg)
    assert bool((out == 12345.0).all())


def test_generic_tile_too_large_for_shared_memory_is_earch():
    """C = 16, pool (4, 4): a 508-position tile of the generic front end needs 16 * 16 * 508 samples of shared memory.
    The configuration is valid (b2cnn_create accepts it, and it runs for short windows: case g-c16-p44-w2430), so a
    window too long for the tile is an architecture limit, B2CNN_EARCH, for forward and features alike, with nothing
    launched and out untouched."""
    ref = O.make_ref(_oarch(BIG_TILE), seed=81)
    assert ref.arch.l_out == 300
    x = tskd_b200.synth.make_windows(2, 16, BIG_TILE[-1], "normal", seed=81, device=DEV)
    m = _model(ref, "relu", random_affine(81))
    rc, out, msg = _raw_forward(m, x, torch.full((2,), 65.0, device=DEV))
    assert rc == capi.EARCH and "shared memory" in msg, (rc, msg)
    assert bool((out == 12345.0).all())
    lib, h = m._ensure_handle()
    feats = torch.full((2, 300), 12345.0, device=DEV)
    rc = lib.b2cnn_features(h, x.data_ptr(), capi.DTYPE_F32, 2, feats.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == capi.EARCH and "shared memory" in capi.last_error()
    assert bool((feats == 12345.0).all())
    with pytest.raises(RuntimeError, match="b2cnn error 2"):
        m.predict(x, 65.0)
