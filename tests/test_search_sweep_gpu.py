"""The brute-force search (csrc/search_topk.cu) and the shard merge against float64, through
tests/gpu_checks.check_search / check_topk_merge (their docstrings state the gates), across the host plan's switches:

  * the cross-partition bound off (m = ceil(k / parts) > 8) with partitions larger than the queue, so 512- and
    2 048-entry queues are cut back mid-scan, in random, all-equal (the tie branch of the cut) and ascending scores;
  * partitions of more than k rows, whose lists of k keys add up to more than the selection kernel stages in shared
    memory (selected from global scratch);
  * k = 256 / 257 (the queue size), 1 024 / 1 025 / 2 049 queries (one launch per 1 024, each with its own output
    offset) with a row offset of 2^33, corpora of 1, 31, 33, 127, 129 rows and N = k = 1 024 (ragged last tile and
    32-score chunk), d = 8, 16, 56, 72 (zero-filled TMA columns), the CITADEL router's shape (Q = 4 100, d = 776);
  * fp16 and bf16 operands, each ranked by the fp32 score and by the fp16-rounded score (--reference_ranking);
  * all-negative and descending scores, and scores that are all zero with mixed signs: -0 and +0 are equal scores,
    so the lower row id (search) or the earlier position (merge) comes first.

Each case names the branch of the plan it is there for, and asserts that _plan, restated from the host code for this
device's SM count, reaches it.  Every case prints the plan it ran.
"""
import pytest

pytestmark = pytest.mark.gpu

CT = 128             # corpus rows per tile
QT = 128             # queries per tile
MAX_QTILES = 8       # query tiles per launch
SEL_SMEM_KEYS = 22528


def _cdiv(a, b):
    return -(-a // b)


def _plan(Q, N, d, k, sms=None):
    """search_topk's host decisions (csrc/search_topk.cu: search_topk, cap_for_k, ws_layout) for `sms` SMs (default:
    this device): the queue size, the 64-column k-blocks and how many of their columns TMA fills with zeros; per
    launch: nb query tiles, parts corpus partitions of tpp tiles, m_track (0 = bound off), the fewest / most rows in a
    partition, and, with the bound off, the keys each query hands to the selection kernel (a partition's queue then
    ends with exactly min(rows, k) keys) and whether they overflow its shared memory."""
    if sms is None:
        from dpr_scale_b200 import _lib
        sms = _lib.load().dprb_num_sms()
    cap = 512 if k <= 256 else 2048
    tiles = _cdiv(N, CT)
    qtiles = _cdiv(Q, QT)
    launches = []
    for qt0 in range(0, qtiles, MAX_QTILES):
        nb = min(MAX_QTILES, qtiles - qt0)
        parts = max(1, min(sms // nb, tiles))
        tpp = _cdiv(tiles, parts)
        parts = _cdiv(tiles, tpp)
        m = _cdiv(k, parts)
        rows = [min(N, (p + 1) * tpp * CT) - p * tpp * CT for p in range(parts)]
        m_track = m if m <= 8 else 0
        keys = sum(min(r, k) for r in rows) if m_track == 0 else None
        launches.append(dict(queries=min(Q - qt0 * QT, nb * QT), nb=nb, parts=parts, tpp=tpp, m_track=m_track,
                             rows=(min(rows), max(rows)), keys=keys,
                             scratch=keys is not None and keys > SEL_SMEM_KEYS))
    kblocks = _cdiv(d, 64)
    return dict(sms=sms, cap=cap, tiles=tiles, kblocks=kblocks, zero_cols=kblocks * 64 - d, launches=launches)


def _all(P, f):
    return all(f(L) for L in P["launches"])


def _cut_without_bound(P):
    """bound off and a partition longer than the queue: every row is queued until the first cut, and the queue is
    cut once it holds more than cap - 32 entries at a 32-score chunk, i.e. when a partition has more than cap rows"""
    return _all(P, lambda L: L["m_track"] == 0 and L["rows"][1] > P["cap"])


F16, BF16 = False, True
SEARCH = [
    # branch, (Q, N, d, k), check_search keyword arguments, what the plan must show
    ("cut-2048-bound-off", (500, 100000, 128, 1024), {}, lambda P: P["cap"] == 2048 and _cut_without_bound(P)),
    ("cut-2048-bound-off-tied", (500, 100000, 128, 1024), {"mode": "constant"},
     lambda P: P["cap"] == 2048 and _cut_without_bound(P)),
    ("cut-2048-bound-off-ascending", (500, 100000, 128, 1024), {"mode": "ascending"},
     lambda P: P["cap"] == 2048 and _cut_without_bound(P)),
    ("cut-512-bound-off", (1024, 50000, 128, 200), {}, lambda P: P["cap"] == 512 and _cut_without_bound(P)),
    ("cut-512-bound-off-tied", (1024, 50000, 128, 200), {"mode": "constant"},
     lambda P: P["cap"] == 512 and _cut_without_bound(P)),
    ("cut-512-bound-off-ascending", (1024, 50000, 128, 200), {"mode": "ascending"},
     lambda P: P["cap"] == 512 and _cut_without_bound(P)),
    ("cut-512-bound-off-f16rank", (1024, 50000, 128, 200), {"reference_ranking": True},
     lambda P: P["cap"] == 512 and _cut_without_bound(P)),
    ("lists-of-k-from-scratch", (200, 80000, 64, 1024), {},
     lambda P: _all(P, lambda L: L["m_track"] == 0 and L["scratch"])),
    ("queue-512-k256", (300, 40000, 128, 256), {}, lambda P: P["cap"] == 512),
    ("queue-2048-k257", (300, 40000, 128, 257), {}, lambda P: P["cap"] == 2048),
    ("one-full-launch-Q1024", (1024, 20000, 64, 16), {"offset": 2 ** 33},
     lambda P: [L["queries"] for L in P["launches"]] == [1024]),
    ("two-launches-Q1025", (1025, 20000, 64, 16), {"offset": 2 ** 33},
     lambda P: [L["queries"] for L in P["launches"]] == [1024, 1]),
    ("three-launches-Q2049", (2049, 20000, 64, 16), {"offset": 2 ** 33},
     lambda P: [L["queries"] for L in P["launches"]] == [1024, 1024, 1]),
    ("N1", (5, 1, 64, 1), {}, lambda P: P["tiles"] == 1),
    ("N31", (5, 31, 64, 10), {}, lambda P: P["tiles"] == 1),
    ("N33", (5, 33, 64, 10), {}, lambda P: P["tiles"] == 1),
    ("N127", (5, 127, 64, 10), {}, lambda P: P["tiles"] == 1),
    ("N129-ragged-second-tile", (5, 129, 64, 10), {}, lambda P: P["tiles"] == 2),
    ("N-equals-k-1024", (3, 1024, 64, 1024), {},
     lambda P: _all(P, lambda L: L["m_track"] == 0 and L["rows"][1] < 1024 and L["keys"] == 1024)),
    ("d8", (100, 10000, 8, 50), {}, lambda P: P["kblocks"] == 1 and P["zero_cols"] == 56),
    ("d16", (100, 10000, 16, 50), {}, lambda P: P["kblocks"] == 1 and P["zero_cols"] == 48),
    ("d56", (100, 10000, 56, 50), {}, lambda P: P["kblocks"] == 1 and P["zero_cols"] == 8),
    ("d72-two-kblocks", (100, 10000, 72, 50), {}, lambda P: P["kblocks"] == 2 and P["zero_cols"] == 56),
    ("router-k1", (4100, 30522, 776, 1), {},
     lambda P: len(P["launches"]) == 5 and P["zero_cols"] > 0 and _all(P, lambda L: L["m_track"] == 1)),
    ("router-k8", (4100, 30522, 776, 8), {},
     lambda P: len(P["launches"]) == 5 and P["zero_cols"] > 0 and _all(P, lambda L: L["m_track"] > 0)),
    ("fp16-bound-on", (300, 20000, 256, 100), {"bf16": F16}, lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("bf16-bound-on", (300, 20000, 256, 100), {"bf16": BF16}, lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("fp16-bound-on-f16rank", (300, 20000, 256, 100), {"bf16": F16, "reference_ranking": True},
     lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("bf16-bound-on-f16rank", (300, 20000, 256, 100), {"bf16": BF16, "reference_ranking": True},
     lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("negative-bound-on", (200, 30000, 128, 100), {"mode": "negative"}, lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("negative-bound-off", (200, 30000, 128, 1000), {"mode": "negative"},
     lambda P: _all(P, lambda L: L["m_track"] == 0)),
    ("descending-bound-on", (64, 20000, 64, 100), {"mode": "descending"},
     lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("descending-bound-off", (64, 20000, 64, 1000), {"mode": "descending"},
     lambda P: _all(P, lambda L: L["m_track"] == 0)),
    ("signed_zero_f16-bound-on", (3, 5000, 64, 100), {"mode": "signed_zero_f16", "reference_ranking": True},
     lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("signed_zero_f16-bound-off", (3, 5000, 64, 1000), {"mode": "signed_zero_f16", "reference_ranking": True},
     lambda P: _all(P, lambda L: L["m_track"] == 0)),
    ("signed_zero_f16-bf16", (3, 5000, 64, 100),
     {"mode": "signed_zero_f16", "reference_ranking": True, "bf16": BF16},
     lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("zero_query-bound-on", (50, 6000, 64, 100), {"mode": "zero_query"}, lambda P: _all(P, lambda L: L["m_track"] > 0)),
    ("zero_query-bound-off", (50, 6000, 64, 1000), {"mode": "zero_query"},
     lambda P: _all(P, lambda L: L["m_track"] == 0)),
    ("zero_query-f16rank", (50, 6000, 64, 100), {"mode": "zero_query", "reference_ranking": True},
     lambda P: _all(P, lambda L: L["m_track"] > 0)),
]


@pytest.mark.parametrize("branch,shape,kw,reaches", SEARCH, ids=[c[0] for c in SEARCH])
def test_search_matches_float64(branch, shape, kw, reaches):
    from tests.gpu_checks import check_search
    Q, N, d, k = shape
    P = _plan(Q, N, d, k)
    print(f"{branch}: Q={Q} N={N} d={d} k={k} queue={P['cap']} kblocks={P['kblocks']} zero_cols={P['zero_cols']} "
          + " | ".join(f"nb={L['nb']} parts={L['parts']} tpp={L['tpp']} m_track={L['m_track']} rows={L['rows']} "
                       f"keys={L['keys']} scratch={L['scratch']}" for L in P["launches"]))
    assert reaches(P), f"{branch}: the plan on {P['sms']} SMs does not reach this branch"
    res = check_search(Q, N, d, k, seed=4000 + Q + N + d + k, **kw)
    print({key: f"{v:.3g}" for key, v in res.items()})


MERGE = [
    # (Q, total, k, signed_zero)
    ("signed_zero", (7, 3000, 500, True)),
    ("signed_zero-smem-overflow", (2, 22529, 1000, True)),
    ("k-equals-total", (9, 1000, 1000, False)),
    ("one-query", (1, 300, 100, False)),
    ("total-22529-smem-overflow", (3, SEL_SMEM_KEYS + 1, 1000, False)),
]


@pytest.mark.parametrize("case,args", MERGE, ids=[c[0] for c in MERGE])
def test_topk_merge_matches_float64(case, args):
    from tests.gpu_checks import check_topk_merge
    Q, total, k, signed_zero = args
    assert k <= total
    check_topk_merge(Q, total, k, seed=5000 + total + k, signed_zero=signed_zero)
