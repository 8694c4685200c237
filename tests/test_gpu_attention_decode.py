"""GPU: single-query attention over indexed key rows (univl_attention_decode_fwd, csrc/attention_decode.cu) against
tests/attn_check.py's fp64 reference with per-element bounds.

Lists of 1 to 1024 keys, scattered and duplicate row indices, one list shared by several queries, an empty list, with
and without list_of_query.  K|V rows no list names hold NaN, so a kernel that read one would fail; the output rows sit
in a sentinel-filled buffer with ldo > 768 whose padding must survive."""
import pytest
import torch

from tests import attn_check as A
from tests.gemm_check import SENT_BF16, SENT_F32, U
from univl_b200 import ops
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 768
COUNTS = [1, 2, 17, 256, 257, 512, 1024, 0, 3]
LD_KV = 2 * H + 64
LD_ROWS = 1024 + 7
LDO = H + 64


class Case:
    def __init__(self, counts, seed, shared=True):
        g = torch.Generator().manual_seed(seed)
        self.counts = counts
        n_lists = len(counts)
        pool = 3 * max(counts) + 100
        table = torch.zeros(n_lists, LD_ROWS, dtype=torch.int32)
        for c, n in enumerate(counts):
            rows = torch.randperm(pool, generator=g)[:n]
            if n >= 17 and c % 2 == 0:
                rows[n // 2:n // 2 + 5] = rows[:5]          # duplicate indices: the same key row listed twice
            table[c, :n] = rows.to(torch.int32)
        listed = torch.zeros(pool, dtype=torch.bool)
        for c, n in enumerate(counts):
            listed[table[c, :n].long()] = True
        kv = torch.full((pool, LD_KV), float("nan"), dtype=torch.bfloat16)
        kv[listed] = (torch.randn(int(listed.sum()), LD_KV, generator=g) * 0.6).to(torch.bfloat16)
        self.kv = kv.to(DEV)
        self.table = table.to(DEV)
        self.n_keys = torch.tensor(counts, dtype=torch.int32, device=DEV)
        # query r reads list r; with `shared`, three more queries read list 3 (256 keys) and one reads list 0
        lists = list(range(n_lists)) + ([3, 3, 3, 0] if shared else [])
        self.lists = lists
        self.loq = torch.tensor(lists, dtype=torch.int32, device=DEV) if shared else None
        self.q = (torch.randn(len(lists), H, generator=g) * 0.6).to(torch.bfloat16).to(DEV)

    def run(self, n_keys=None):
        n_q = self.q.shape[0]
        obuf = torch.full((n_q + 3, LDO), SENT_BF16, dtype=torch.bfloat16, device=DEV)
        lbuf = torch.full((n_q + 3, A.HEADS), SENT_F32, dtype=torch.float32, device=DEV)
        ops.attention_decode_fwd(self.q, self.kv, self.table, self.n_keys if n_keys is None else n_keys, self.loq,
                                 out=obuf[:n_q, :H], lse=lbuf)
        return obuf, lbuf

    def reference(self, r):
        c = self.lists[r]
        n = self.counts[c]
        rows = self.table[c, :n].long()
        k, v = self.kv[rows, :H], self.kv[rows, H:2 * H]
        ref = A.reference(self.q[r:r + 1], k, v, 1, 1, n, torch.ones(1, n, dtype=torch.int64, device=DEV),
                          kind="long", want_p=True)
        # kind "long" budgets ceil(n / 64) online-softmax rescales; the decode kernel rescales a warp's partials once
        # per 4-key chunk (a warp reads keys w, w + 8, ...: ceil(n / 32) chunks) and once more in the warp merge.  Each
        # extra rescale errs by EXP_REL + 2U relative, on the normaliser and on every P-weighted term of the context.
        extra = (-(-n // 32) + 1 - (-(-n // 64))) * (A.EXP_REL + 2 * U)
        pv = A._unheads(ref["p"] @ A._heads(v, 1, n).abs())
        ref["b_o"] = ref["b_o"] + extra * pv
        ref["b_lse"] = ref["b_lse"] + extra
        return ref


@pytest.mark.parametrize("shared", [True, False], ids=["list_of_query", "identity"])
def test_decode_attention_against_fp64(shared):
    case = Case(COUNTS, seed=5 + shared, shared=shared)
    obuf, lbuf = case.run()
    n_q = case.q.shape[0]
    for r in range(n_q):
        n = case.counts[case.lists[r]]
        if n == 0:   # an empty list writes nothing
            assert bool((obuf[r] == SENT_BF16).all()) and bool((lbuf[r] == SENT_F32).all())
            continue
        ref = case.reference(r)
        A.check_fwd(obuf[r:r + 1, :H], lbuf[r], ref, "decode query %d (%d keys)" % (r, n))
    assert bool((obuf[:, H:] == SENT_BF16).all()) and bool((obuf[n_q:] == SENT_BF16).all())
    assert bool((lbuf[n_q:] == SENT_F32).all())
    # repeated launches, and launches beside a reserved-SM collective, give the same bits
    o2, l2 = case.run()
    assert torch.equal(o2, obuf) and torch.equal(l2, lbuf)
    rt.reserve_sms(40)
    try:
        o3, l3 = case.run()
    finally:
        rt.reserve_sms(0)
    assert torch.equal(o3, obuf) and torch.equal(l3, lbuf)


def test_checker_rejects_a_list_missing_its_last_key():
    case = Case(COUNTS, seed=11)
    for c in (1, 2):   # 2 and 17 keys
        short = case.n_keys.clone()
        short[c] -= 1
        obuf, lbuf = case.run(short)
        ref = case.reference(c)
        with pytest.raises(AssertionError):
            A.check_fwd(obuf[c:c + 1, :H], lbuf[c], ref, "list %d without its last key" % c)
        obuf, lbuf = case.run()
        A.check_fwd(obuf[c:c + 1, :H], lbuf[c], ref, "list %d" % c)


def test_bad_arguments_are_rejected():
    case = Case([4, 9], seed=1, shared=False)
    with pytest.raises(RuntimeError, match="heads must be 12"):
        rt.call("univl_attention_decode_fwd", case.q.data_ptr(), H, case.kv.data_ptr(), LD_KV, case.table.data_ptr(),
                LD_ROWS, case.n_keys.data_ptr(), None, 2, 8, case.q.data_ptr(), H, None, A.SCALE)
    with pytest.raises(RuntimeError, match="row stride >= 1536"):
        ops.attention_decode_fwd(case.q, case.kv[:, :H].contiguous(), case.table, case.n_keys)
    with pytest.raises(RuntimeError, match="int32"):
        ops.attention_decode_fwd(case.q, case.kv, case.table.long(), case.n_keys)
