"""CPU: the FP8 entry points (include/univl_b200.h) reject bad arguments before touching a device, with errors that
name the entry point; the evaluation precision switch rejects unknown values."""
import pytest

from univl_b200 import lib


def _fails(name, *args, match):
    with pytest.raises(RuntimeError) as e:
        lib.call(name, *args)
    msg = str(e.value)
    assert name in msg.split(":", 1)[1], msg  # named in the library's message, not only by the wrapper
    assert match in msg, msg


P = 1 << 20  # a 16-byte aligned stand-in address: validation never dereferences it


def test_quantize_rows_arguments():
    q = "univl_quantize_e4m3_rows"
    _fails(q, P, 768, P, 768, P, 0, 768, None, match="empty")
    _fails(q, P, 768, P, 768, P, 4, 700, None, match="multiple of 128")
    _fails(q, None, 768, P, 768, P, 4, 768, None, match="null")
    _fails(q, P, 640, P, 768, P, 4, 768, None, match="ldx/ldq")
    _fails(q, P, 770, P, 768, P, 4, 768, None, match="ldx/ldq")
    _fails(q, P + 2, 768, P, 768, P, 4, 768, None, match="aligned")


def test_quantize_blocks_arguments():
    q = "univl_quantize_e4m3_blocks"
    _fails(q, P, 768, P, 768, P, 768, 0, None, match="empty")
    _fails(q, P, 768, P, 768, P, 700, 768, None, match="multiples of 128")
    _fails(q, P, 768, P, 768, P, 768, 700, None, match="multiples of 128")
    _fails(q, P, 768, None, 768, P, 768, 768, None, match="null")
    _fails(q, P, 766, P, 768, P, 768, 768, None, match="ldw/ldq")
    _fails(q, P + 4, 768, P, 768, P, 768, 768, None, match="aligned")


def _gemm(A=P, lda=768, sa=P, B=P, ldb=768, sb=P, M=256, N=768, K=768, epi=0, bias=P, out=P, ldo=768, so=P):
    return ("univl_gemm_fp8", A, lda, sa, B, ldb, sb, M, N, K, epi, bias, out, ldo, so, None)


def test_gemm_fp8_arguments():
    cases = [
        (dict(M=0), "empty"),
        (dict(K=700, lda=704, ldb=704), "K=700 must be a multiple of 128"),
        (dict(N=700, ldo=704), "N=700 must be a multiple of 128"),
        (dict(epi=2), "unknown epilogue"),
        (dict(sa=None), "null"),
        (dict(bias=None), "null"),
        (dict(lda=640), "lda/ldb"),
        (dict(ldb=776), "lda/ldb"),
        (dict(A=P + 8), "16-byte aligned"),
        (dict(ldo=640), "ldo"),
        (dict(epi=1, so=None), "out_scale"),
        (dict(epi=1, ldo=776), "ldo a multiple of 16"),
    ]
    for kw, match in cases:
        name, *args = _gemm(**kw)
        _fails(name, *args, match=match)


def test_eval_precision_switch(monkeypatch):
    from univl_b200.modules import modeling
    monkeypatch.delenv("UNIVL_EVAL_PRECISION", raising=False)
    assert modeling.eval_precision() == "bf16"
    for v in ("bf16", "fp8"):
        monkeypatch.setenv("UNIVL_EVAL_PRECISION", v)
        assert modeling.eval_precision() == v
    for v in ("", "FP8", "e4m3", "fp16"):
        monkeypatch.setenv("UNIVL_EVAL_PRECISION", v)
        with pytest.raises(ValueError, match="UNIVL_EVAL_PRECISION"):
            modeling.eval_precision()
