"""CPU-only checks of the pair attention entry (univl_attention_pair_fwd): the library exports it, the header
declares it, and bad arguments are rejected with a message before any launch, so no GPU is needed."""
import pytest

from univl_b200 import build, lib
from univl_b200.modules import modeling

P = 16  # any non-null, 16-byte aligned value: the argument checks reject before anything is dereferenced


def _pair(Na=4, Wa=48, Nb=5, Fb=48, heads=12, Sq=96, ld=2304, ldb=2304, qb=P, mask_a=P, mask_b=P, align=0):
    lib.call("univl_attention_pair_fwd", P + align, ld, P, ld, P, ld, qb, ldb, P, ldb, P, ldb, P, 768, None, mask_a,
             mask_b, Na, Wa, Nb, Fb, heads, Sq, 0.125, None)


def test_pair_entry_is_exported_and_declared():
    import ctypes
    handle = ctypes.CDLL(build.build())
    assert hasattr(handle, "univl_attention_pair_fwd")
    assert "univl_attention_pair_fwd" in lib.parse_header()


def test_pair_entry_accepts_good_arguments_without_work():
    _pair(Na=0)  # no pairs: validated, nothing launched


@pytest.mark.parametrize("kwargs, message", [
    (dict(heads=8), r"heads must be 12"),
    (dict(Wa=1000, Fb=25, Sq=1025), r"S <= 1024"),
    (dict(Wa=0), r"bad source shape"),
    (dict(Nb=0), r"bad source shape"),
    (dict(Fb=-1), r"bad source shape"),
    (dict(Sq=0), r"Sq must be 1 or Wa \+ Fb = 96"),
    (dict(Sq=48), r"Sq must be 1 or Wa \+ Fb = 96"),
    (dict(Na=50000, Nb=50000), r"too many pairs"),
    (dict(ld=2308), r"multiples of 8"),
    (dict(ldb=2308), r"second-source row strides must be multiples of 8"),
    (dict(align=8), r"16-byte aligned"),
    (dict(qb=P + 8), r"second-source q/k/v must be 16-byte aligned"),
    (dict(qb=None), r"null second-source q/k/v"),
    (dict(mask_b=None), r"both mask parts are needed when Fb > 0"),
    (dict(mask_a=None), r"both mask parts are needed when Fb > 0"),
])
def test_pair_entry_rejects_bad_arguments(kwargs, message):
    with pytest.raises(RuntimeError, match=message):
        _pair(**kwargs)


@pytest.mark.parametrize("Nt, Nv, S, budget", [(7, 5, 10, 60), (3500, 3500, 96, 1 << 18), (1, 9, 300, 1),
                                               (64, 64, 96, 1 << 40)])
def test_eval_tiles_stay_in_budget_and_cover(Nt, Nv, S, budget):
    bt, bv = modeling._eval_tile(Nt, Nv, S, budget)
    assert 1 <= bt <= Nt and 1 <= bv <= Nv
    assert bt * bv * S <= max(budget, S)
