"""CPU-only checks of the key-tiled attention entries (univl_attention_long_fwd / _bwd): the library exports them, and
bad arguments are rejected with a message before any launch, so no GPU is needed."""
import pytest

from univl_b200 import build, lib, ops

P = 16  # any non-null, 16-byte aligned value: the argument checks reject before anything is dereferenced


def _fwd(Sq=300, Sk=300, heads=12, ldq=768, n_seq=1):
    lib.call("univl_attention_long_fwd", P, ldq, P, 768, P, 768, P, 768, None, None, None, 0, 0, 0, 0, n_seq, heads,
             Sq, Sk, 0, 0.125, 0.0, 0, 0, None)


def _bwd(Sq=300, Sk=300, heads=12, ldq=768, rng_layout=0, lddo=768, dbias=(None, None, None)):
    lib.call("univl_attention_long_bwd", P, ldq, P, 768, P, 768, P, 768, P, P, lddo, P, 768, P, 768, P, 768, None,
             None, 0, 0, 0, 0, 1, heads, Sq, Sk, 0, 0.125, 0.0, 0, 0, rng_layout, *dbias, None)


def test_long_entries_are_exported():
    import ctypes
    handle = ctypes.CDLL(build.build())
    for name in ("univl_attention_long_fwd", "univl_attention_long_bwd"):
        assert hasattr(handle, name)
        assert name in lib.parse_header()


@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_long_entries_reject_bad_arguments(call):
    with pytest.raises(RuntimeError, match=r"S <= 1024"):
        call(Sq=1025, Sk=300)
    with pytest.raises(RuntimeError, match=r"S <= 1024"):
        call(Sq=1, Sk=2048)
    with pytest.raises(RuntimeError, match=r"unsupported shape"):
        call(Sq=0, Sk=300)
    with pytest.raises(RuntimeError, match=r"heads must be 12"):
        call(heads=8)
    with pytest.raises(RuntimeError, match=r"multiples of 8"):
        call(ldq=770)


def test_long_bwd_rejects_row_major_dropout_layout_and_bad_strides():
    with pytest.raises(RuntimeError, match=r"rng_layout must be 0"):
        _bwd(rng_layout=1)
    with pytest.raises(RuntimeError, match=r"bad strides"):
        _bwd(lddo=770)
    with pytest.raises(RuntimeError, match=r"all set or all null"):
        _bwd(dbias=(P, None, None))


def test_dispatch_by_length():
    """up to 256 tokens the existing entries; above, in either dimension, the key-tiled ones"""
    assert ops._attention_entry("fwd", 256, 256) == "univl_attention_fwd"
    assert ops._attention_entry("bwd", 1, 256) == "univl_attention_bwd"
    assert ops._attention_entry("fwd", 257, 257) == "univl_attention_long_fwd"
    assert ops._attention_entry("fwd", 1, 1024) == "univl_attention_long_fwd"
    assert ops._attention_entry("bwd", 300, 16) == "univl_attention_long_bwd"
