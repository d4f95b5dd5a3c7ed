"""Architecture description of the reference's ``MyCNN`` (bin/models.py:6-20) and its older
revisions (bin/explore_torch copy.ipynb:189-277), plus the state_dict key contract."""
from __future__ import annotations

from dataclasses import dataclass, replace
from typing import Dict, Mapping, Tuple

ACT_TANH, ACT_RELU, ACT_IDENTITY = 0, 1, 2
_ACT_NAMES = {"tanh": ACT_TANH, "relu": ACT_RELU, "identity": ACT_IDENTITY}

# Tensors the forward pass uses, in packed-blob order (include/b2cnn.h).
BLOB_KEYS: Tuple[str, ...] = (
    "conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias",
    "lstm.weight_ih_l0", "lstm.weight_hh_l0", "lstm.bias_ih_l0", "lstm.bias_hh_l0",
    "lstm.weight_ih_l1", "lstm.weight_hh_l1", "lstm.bias_ih_l1", "lstm.bias_hh_l1",
    "out.weight", "out.bias")
# Constructed by the reference but never used in forward (bin/models.py:13,18,20): kept as
# inert entries so state_dict()/load_state_dict() round-trip the reference's key set.
INERT_KEYS: Tuple[str, ...] = ("out1.weight", "out1.bias", "out2.weight", "out2.bias",
                               "age_fn.weight", "age_fn.bias")


@dataclass(frozen=True)
class ArchConfig:
    in_channels: int = 10        # bin/models.py:10
    k1: int = 10                 # bin/models.py:10
    k2: int = 5                  # bin/models.py:11
    pool_k: int = 3              # bin/models.py:12
    pool_s: int = 2              # bin/models.py:12
    window: int = 120            # config.cfg:23 (WINDOWSIZE)
    age_coef: float = 1e-8       # bin/models.py:32
    act: str = "tanh"            # bin/models.py:23,26
    affine: bool = False         # optional folded eval-BatchNorm after each conv
    c_mid: int = 4
    hidden: int = 16
    layers: int = 2

    @property
    def l1(self) -> int:
        return self.window - self.k1 + 1

    @property
    def p1(self) -> int:
        return (self.l1 - self.pool_k) // self.pool_s + 1

    @property
    def l2(self) -> int:
        return self.p1 - self.k2 + 1

    @property
    def l_out(self) -> int:
        """MAGICNUM (bin/models.py:8): the LSTM input size == features per window."""
        return (self.l2 - self.pool_k) // self.pool_s + 1

    @property
    def receptive_field(self) -> int:
        """Samples one feature reads; features start pool_s ** 2 samples apart, so l_out = (window - R) // pool_s ** 2 + 1."""
        return self.pool_s * (self.pool_k + self.k2 - 2) + self.pool_k + self.k1 - 1

    @property
    def act_id(self) -> int:
        return _ACT_NAMES[self.act]

    def with_shape(self, in_channels: int, window: int) -> "ArchConfig":
        return replace(self, in_channels=in_channels, window=window)

    def param_shapes(self) -> Dict[str, Tuple[int, ...]]:
        L, H, G = self.l_out, self.hidden, 4 * self.hidden
        return {
            "conv1.weight": (self.c_mid, self.in_channels, self.k1), "conv1.bias": (self.c_mid,),
            "conv2.weight": (1, self.c_mid, self.k2), "conv2.bias": (1,),
            "lstm.weight_ih_l0": (G, L), "lstm.weight_hh_l0": (G, H),
            "lstm.bias_ih_l0": (G,), "lstm.bias_hh_l0": (G,),
            "lstm.weight_ih_l1": (G, H), "lstm.weight_hh_l1": (G, H),
            "lstm.bias_ih_l1": (G,), "lstm.bias_hh_l1": (G,),
            "out.weight": (1, H), "out.bias": (1,),
        }


# MyCNN5 == bin/models.py as shipped; MyCNN2/3/4 == older revision (k1=5, pool(2,2)); their
# age coefficient at save time is unknown (1e-4 in explore_torch copy.ipynb:259, 1e-8 in
# models.py:32) -> a constructor parameter, default per the notebook revision.
ARCH_PRESETS = {
    "mycnn5": ArchConfig(),
    "mycnn4": ArchConfig(in_channels=10, k1=5, pool_k=2, pool_s=2, age_coef=1e-4),
    "mycnn3": ArchConfig(in_channels=7, k1=5, pool_k=2, pool_s=2, age_coef=1e-4),
    "mycnn2": ArchConfig(in_channels=7, k1=5, pool_k=2, pool_s=2, age_coef=1e-4),
}


def arch_from_state_dict(sd: Mapping[str, "object"], window: int | None = None,
                         pool: Tuple[int, int] | None = None, age_coef: float | None = None,
                         act: str = "tanh") -> ArchConfig:
    """Infer the architecture from tensor shapes.  The pool geometry is not in a state_dict:
    it is taken from ``pool`` or solved from lstm.weight_ih_l0's input size among the two
    geometries the reference ever used ((3,2) and (2,2))."""
    c_mid, c_in, k1 = tuple(sd["conv1.weight"].shape)
    k2 = int(sd["conv2.weight"].shape[-1])
    L = int(sd["lstm.weight_ih_l0"].shape[1])
    cands = [pool] if pool else [(3, 2), (2, 2)]
    if window is None:
        # smallest window consistent with L for each candidate geometry; the reference's is 120
        for pk, ps in cands:
            a = ArchConfig(in_channels=c_in, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=120, act=act)
            if a.l_out == L:
                window = 120
                break
    if window is None:
        raise ValueError("cannot infer the window length from the state_dict; pass window=")
    for pk, ps in cands:
        a = ArchConfig(in_channels=c_in, k1=k1, k2=k2, pool_k=pk, pool_s=ps, window=window, act=act,
                       c_mid=c_mid)
        if a.l1 >= pk and a.l2 >= pk and a.l_out == L:
            if age_coef is None:
                age_coef = 1e-8 if (k1, pk, ps) == (10, 3, 2) else 1e-4
            return replace(a, age_coef=age_coef)
    raise ValueError(f"no pool geometry maps window={window} to lstm input size {L}")
