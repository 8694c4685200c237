"""CPU: the fused vocabulary cross-entropy entry points (include/univl_b200.h) reject bad arguments before touching a
device, with errors that name the entry point; the UNIVL_VOCAB_LOSS switch rejects unknown values."""
import pytest

from univl_b200 import lib

P = 1 << 20  # a 16-byte aligned stand-in address: validation never dereferences it


def _fails(name, *args, match):
    with pytest.raises(RuntimeError) as e:
        lib.call(name, *args)
    msg = str(e.value)
    assert name in msg.split(":", 1)[1], msg  # named in the library's message, not only by the wrapper
    assert match in msg, msg


def _fwd(x=P, ldx=768, w=P, ldw=768, bias=P, labels=P, lse=P, sc=P, loss=P, ws=P, ws_bytes=1 << 30, T=256,
         V=30522, K=768, groups=1):
    return ("univl_vocab_xent_fwd", x, ldx, w, ldw, bias, labels, lse, sc, loss, ws, ws_bytes, T, V, K, groups, None)


def _bwd(x=P, ldx=768, w=P, ldw=768, bias=P, labels=P, lse=P, sc=P, g=P, dl=P, ld_d=30528, T=256, V=30522, K=768,
         groups=1):
    return ("univl_vocab_xent_bwd", x, ldx, w, ldw, bias, labels, lse, sc, g, dl, ld_d, T, V, K, groups, None)


COMMON = [
    (dict(T=0), "empty"),
    (dict(V=0), "empty"),
    (dict(x=None), "null"),
    (dict(labels=None), "null"),
    (dict(ldx=700), "ldx/ldw"),
    (dict(ldw=776 - 4), "ldx/ldw"),
    (dict(w=P + 8), "16-byte aligned"),
    (dict(groups=3), "groups must divide"),
    (dict(groups=0), "groups must divide"),
]


def test_vocab_xent_fwd_arguments():
    for kw, match in COMMON + [(dict(loss=None), "null"), (dict(ws=None), "null"), (dict(ws=P + 4), "aligned"),
                               (dict(ws_bytes=1024), "univl_vocab_xent_workspace")]:
        name, *args = _fwd(**kw)
        _fails(name, *args, match=match)


def test_vocab_xent_bwd_arguments():
    for kw, match in COMMON + [(dict(dl=None), "null"), (dict(ld_d=30520), "ld_d"), (dict(ld_d=30529), "ld_d"),
                               (dict(ld_d=30720), "ld_d"), (dict(dl=P + 2), "ld_d")]:
        name, *args = _bwd(**kw)
        _fails(name, *args, match=match)


def vx_chunks(T, V):
    """(chunks, 128-column tiles per chunk) of the fused vocabulary cross-entropy (vx_plan in csrc/gemm_wgmma.cu)"""
    m, n = -(-T // 128), -(-V // 128)
    best = None
    for c in range(1, n + 1):
        ct = -(-n // c)
        if ct < 8 and c > 1:
            break
        if c > 1 and ct == -(-n // (c - 1)):
            continue
        chunks = -(-n // ct)
        cost = -(-(m * chunks) // 132) * ct
        if best is None or cost < best[0]:
            best = (cost, chunks, ct)
    return best[1], best[2]


def test_vocab_xent_workspace():
    ws = lib.load().univl_vocab_xent_workspace
    # one 16-byte record per row and vocabulary chunk, then one float per row, padded to 16 bytes
    assert vx_chunks(4096, 30522) == (4, 60)     # 32 row tiles x 4 chunks: one round of work items on 132 SMs
    assert vx_chunks(17280, 30522) == (30, 8)
    assert vx_chunks(1, 257) == (1, 3)
    for T, V in ((4096, 30522), (17280, 30522), (1, 257), (127, 1000), (384, 30522)):
        assert ws(T, V) == T * vx_chunks(T, V)[0] * 16 + -(-T * 4 // 16) * 16, (T, V)
    assert ws(0, 30522) < 0
    assert ws(1 << 30, 30522) < 0                # over 2 GiB


def test_vocab_loss_switch(monkeypatch):
    from univl_b200 import ops
    monkeypatch.delenv("UNIVL_VOCAB_LOSS", raising=False)
    assert ops.vocab_loss_mode() == "logits"
    for v in ("logits", "fused"):
        monkeypatch.setenv("UNIVL_VOCAB_LOSS", v)
        assert ops.vocab_loss_mode() == v
    for v in ("", "FUSED", "fp32", "1"):
        monkeypatch.setenv("UNIVL_VOCAB_LOSS", v)
        with pytest.raises(ValueError, match="UNIVL_VOCAB_LOSS"):
            ops.vocab_loss_mode()
