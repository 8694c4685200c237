"""GPU: the variable-length attention forward (univl_attention_varlen_fwd) and the packed row gather
(univl_gather_rows_varlen) of packed pair evaluation, against tests/attn_check.py's fp64 reference with per-element
bounds (no dropout, no mask: every key is real).

Both row addressings (pair: by index from two sources; packed: back to back), every query row and token 0 only, and
sequences of 1 to 1024 keys mixed in one launch on either side of the 256-key boundary between attention.cu's and
attention_long.cu's kernels.  Source rows no sequence indexes hold NaN, so a kernel that read one would fail; output
rows and columns outside the packed ranges hold sentinels that must survive."""
import pytest
import torch

from tests import attn_check as A
from tests.gemm_check import SENT_BF16, SENT_F32
from univl_b200 import ops
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 768
SHORT = [1, 5, 16, 17, 33, 48, 96, 100, 128, 129, 200, 255, 256, 3]
LONG = [1, 2, 15, 17, 64, 65, 255, 256, 257, 300, 511, 640, 1023, 1024, 40]
# longest 97..128 keys: attention.cu's register-resident score row of 8 key blocks (NKB = 8); SHORT runs its two-pass
# variant (NKB = 0), and MID's shorter sequences the 3- and 6-block rows' lengths
MID = [1, 7, 16, 33, 48, 64, 97, 100, 113, 120]


def _split(lens, g):
    """(len_a, len_b) per sequence: random splits, including all-a (a fully padded second source) and all-b"""
    la = []
    for k, n in enumerate(lens):
        if k % 5 == 0:
            la.append(n)
        elif k % 7 == 3:
            la.append(0)
        else:
            la.append(int(torch.randint(0, n + 1, (1,), generator=g)))
    return la, [n - a for n, a in zip(lens, la)]


def _i32(x):
    return torch.tensor(x, dtype=torch.int32, device=DEV)


class Case:
    """one launch's sequences with their sources; materialise(p) gives sequence p's q / k / v rows"""

    def __init__(self, lens, pair, seed):
        g = torch.Generator().manual_seed(seed)
        self.lens, self.pair = lens, pair
        n = len(lens)
        cu = [0]
        for s in lens:
            cu.append(cu[-1] + s)
        self.total = cu[-1]
        self.max_sk = max(lens)
        if pair:
            la, lb = _split(lens, g)
            NA, NB = sum(la) + 37, sum(lb) + 29
            self.a = torch.full((NA, 3 * H), float("nan"), dtype=torch.bfloat16)
            self.b = torch.full((NB, 3 * H), float("nan"), dtype=torch.bfloat16)
            ra = torch.randperm(NA, generator=g)[:sum(la)]  # scattered rows, each indexed once
            rb = torch.randperm(NB, generator=g)[:sum(lb)]
            self.a[ra] = (torch.randn(len(ra), 3 * H, generator=g) * 0.6).to(torch.bfloat16)
            self.b[rb] = (torch.randn(len(rb), 3 * H, generator=g) * 0.6).to(torch.bfloat16)
            self.a, self.b = self.a.to(DEV), self.b.to(DEV)
            sa, sb = [0], [0]
            for x, y in zip(la, lb):
                sa.append(sa[-1] + x)
                sb.append(sb[-1] + y)
            self.rows = [(ra[sa[p]:sa[p + 1]], rb[sb[p]:sb[p + 1]]) for p in range(n)]
            self.seqs = ops.VarlenSeqs(_i32(cu), self.total, self.max_sk, _i32(ra.tolist()), _i32(rb.tolist()),
                                       _i32(sa[:-1]), _i32(sb[:-1]), _i32(la))
        else:
            self.a = torch.full((self.total + 11, 3 * H), float("nan"), dtype=torch.bfloat16)
            self.a[:self.total] = (torch.randn(self.total, 3 * H, generator=g) * 0.6).to(torch.bfloat16)
            self.a = self.a.to(DEV)
            self.q0 = (torch.randn(n, H, generator=g) * 0.6).to(torch.bfloat16).to(DEV)  # packed token-0 queries
            self.seqs = ops.VarlenSeqs(_i32(cu), self.total, self.max_sk)
        self.cu = cu

    def materialise(self, p):
        if self.pair:
            ia, ib = self.rows[p]
            return torch.cat([self.a[ia.to(DEV)], self.b[ib.to(DEV)]])
        return self.a[self.cu[p]:self.cu[p + 1]]

    def run(self, q_first, ldo=H + 64, extra_rows=5, seqs=None):
        """-> (o buffer, lse buffer, rows) with sentinel padding around the [rows, H] / [rows, 12] results"""
        seqs = seqs or self.seqs
        rows = seqs.n_seq if q_first else seqs.total
        obuf = torch.full((rows + extra_rows, ldo), SENT_BF16, dtype=torch.bfloat16, device=DEV)
        lbuf = torch.full((rows + extra_rows, A.HEADS), SENT_F32, dtype=torch.float32, device=DEV)
        a = self.a
        q = self.q0 if (q_first and not self.pair) else a[:, :H]
        b = self.b if self.pair else None
        rt.call("univl_attention_varlen_fwd", q.data_ptr(), q.stride(0), a[:, H:].data_ptr(), a.stride(0),
                a[:, 2 * H:].data_ptr(), a.stride(0), rt.ptr(b), b.stride(0) if self.pair else 0,
                b[:, H:].data_ptr() if self.pair else None, b.stride(0) if self.pair else 0,
                b[:, 2 * H:].data_ptr() if self.pair else None, b.stride(0) if self.pair else 0,
                *seqs.index_args(), seqs.n_seq, seqs.max_sk, A.HEADS, int(q_first), obuf.data_ptr(), obuf.stride(0),
                lbuf.data_ptr(), A.SCALE)
        return obuf, lbuf, rows


def _check(case, q_first, obuf, lbuf, what):
    kind = "short" if case.max_sk <= 256 else "long"
    for p, Sk in enumerate(case.lens):
        seq = case.materialise(p)
        q = seq[:, :H]
        if q_first:
            q = case.q0[p:p + 1] if not case.pair else q[:1]
        Sq = q.shape[0]
        ref = A.reference(q, seq[:, H:2 * H], seq[:, 2 * H:], 1, Sq, Sk, torch.ones(1, Sk, dtype=torch.int64,
                                                                                     device=DEV), kind=kind)
        r0 = p if q_first else case.cu[p]
        o = obuf[r0:r0 + Sq, :H]
        lse = lbuf[r0:r0 + Sq].t().reshape(-1)  # [rows, heads] -> reference's [heads, Sq]
        A.check_fwd(o, lse, ref, "%s seq %d (Sk %d)" % (what, p, Sk))


@pytest.mark.parametrize("lens", [MID, SHORT, LONG], ids=["mid", "short", "long"])
@pytest.mark.parametrize("pair", [True, False], ids=["pair", "packed"])
@pytest.mark.parametrize("q_first", [False, True], ids=["all", "first"])
def test_varlen_attention_against_fp64(lens, pair, q_first):
    case = Case(lens, pair, seed=len(lens) + 2 * pair + q_first)
    obuf, lbuf, rows = case.run(q_first)
    _check(case, q_first, obuf, lbuf, "varlen %s %s" % ("pair" if pair else "packed", "first" if q_first else "all"))
    # outside the packed ranges: padding columns and rows past the result untouched
    assert bool((obuf[:rows, H:] == SENT_BF16).all()) and bool((obuf[rows:] == SENT_BF16).all())
    assert bool((lbuf[rows:] == SENT_F32).all())
    # repeated launches, and launches beside a reserved-SM collective, give the same bits
    o2, l2, _ = case.run(q_first)
    assert torch.equal(o2, obuf) and torch.equal(l2, lbuf)
    rt.reserve_sms(40)
    try:
        o3, l3, _ = case.run(q_first)
    finally:
        rt.reserve_sms(0)
    assert torch.equal(o3, obuf) and torch.equal(l3, lbuf)


def test_checker_rejects_a_result_with_one_dropped_key():
    """the same launch with sequence 3's last key left out fails the bounds of the full sequence"""
    case = Case(SHORT, True, seed=9)
    cu = list(case.cu)
    for p in range(4, len(cu)):
        cu[p] -= 1  # sequence 3 (17 keys) loses its last key; the later ones keep theirs (shifted by one row)
    la = case.seqs.len_a.clone()
    la[3] = min(int(la[3]), case.lens[3] - 1)
    dropped = ops.VarlenSeqs(_i32(cu), case.total - 1, case.max_sk, case.seqs.idx_a, case.seqs.idx_b,
                             case.seqs.start_a, case.seqs.start_b, la)
    obuf, lbuf, _ = case.run(True, seqs=dropped)
    seq = case.materialise(3)
    ref = A.reference(seq[:1, :H], seq[:, H:2 * H], seq[:, 2 * H:], 1, 1, 17,
                      torch.ones(1, 17, dtype=torch.int64, device=DEV))
    with pytest.raises(AssertionError):
        A.check_fwd(obuf[3:4, :H], lbuf[3:4].t().reshape(-1), ref, "one dropped key")
    # and the untouched launch passes the same check
    obuf, lbuf, _ = case.run(True)
    A.check_fwd(obuf[3:4, :H], lbuf[3:4].t().reshape(-1), ref, "all keys")


@pytest.mark.parametrize("pair", [True, False], ids=["pair", "packed"])
@pytest.mark.parametrize("q_first", [False, True], ids=["all", "first"])
def test_gather_rows_in_packed_order(pair, q_first):
    case = Case(LONG, pair, seed=21)
    n = case.seqs.n_seq
    rows = n if q_first else case.total
    ld = 3 * H + 64
    buf = torch.full((rows + 4, ld), SENT_BF16, dtype=torch.bfloat16, device=DEV)
    b = case.b if pair else None
    rt.call("univl_gather_rows_varlen", case.a.data_ptr(), case.a.stride(0), rt.ptr(b), b.stride(0) if pair else 0,
            *case.seqs.index_args(), n, int(q_first), 3 * H, buf.data_ptr(), buf.stride(0))
    want = torch.cat([case.materialise(p)[:1] if q_first else case.materialise(p) for p in range(n)])
    assert torch.equal(buf[:rows, :3 * H], want)
    assert bool((buf[:rows, 3 * H:] == SENT_BF16).all()) and bool((buf[rows:] == SENT_BF16).all())
    got = ops.gather_rows_varlen(case.a, b, case.seqs, q_first)
    assert torch.equal(got, want)


def test_bad_arguments_are_rejected():
    case = Case([4, 9], True, seed=1)
    s = case.seqs
    with pytest.raises(RuntimeError, match="pair addressing needs"):
        ops.attention_varlen_fwd(case.a[:, :H], case.a[:, H:2 * H], case.a[:, 2 * H:],
                                 ops.VarlenSeqs(s.cu, s.total, s.max_sk, s.idx_a, None, s.start_a, s.start_b, s.len_a),
                                 False, case.b[:, :H], case.b[:, H:2 * H], case.b[:, 2 * H:])
    with pytest.raises(RuntimeError, match="unsupported shape"):
        ops.attention_varlen_fwd(case.a[:, :H], case.a[:, H:2 * H], case.a[:, 2 * H:],
                                 ops.VarlenSeqs(s.cu, s.total, 1025, s.idx_a, s.idx_b, s.start_a, s.start_b, s.len_a),
                                 False, case.b[:, :H], case.b[:, H:2 * H], case.b[:, 2 * H:])
    with pytest.raises(RuntimeError, match="cols must be"):
        rt.call("univl_gather_rows_varlen", case.a.data_ptr(), case.a.stride(0), case.b.data_ptr(), case.b.stride(0),
                *s.index_args(), s.n_seq, 0, 12, case.a.data_ptr(), case.a.stride(0))
