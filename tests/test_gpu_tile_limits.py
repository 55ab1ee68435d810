"""The tile path's shared-memory limits as tested boundaries (csrc/bigclam_tile.cuh TlWarp::run).

A tile runs on the tile path only if it fits the warp's buffers; otherwise the same warp redoes its nodes on the general
path.  For each of the six checks (tests/tile_twin.py) a graph is built with one tile exactly AT the limit (it must run on
the tile path) and one tile ONE PAST it (it must fall back at that check), every other quantity of the two below its own
limit, between ordinary tiles.  The tile counters of the first step must equal the model's prediction exactly, and three
steps must match the oracle.  The cut is pinned with BIGCLAM_TILE_EDGES=32 (no re-cut), so it depends on the degrees only.

Layout of every graph: five groups of 8 nodes of degree 4 (ordinary, AT, ordinary, PAST, ordinary; 32 edges each: one
tile per group), each node with 4 leaves of its own (degree 1, tiles of 8 leaves), then 3 isolated nodes with empty rows
(a tile of its own: no edges, nothing staged).  Component 0 is in every other row, at 0.1: an edge whose rows share
nothing else has x = 0.01 and a weight 1 / (1 - p) of about 100, so a node's gradient is far above 0 on a component only
its neighbours have.  sumF is the column sums of F0 plus 1 (so that it stays clear of 0, as the kernels assume, even
where a column empties), plus 1e5 on the DEAD components: there the gradient is far below 0 wherever the node's own row
is 0, and the component is inactive.

A step launches two step kernels: the step itself and the next call's, speculatively (bigclam_step); the counters after
the first step cover both, so the model predicts the second one from the state the first left (read back from the GPU)."""
import numpy as np
import pytest

import tile_twin as TW
from test_gpu_parity import _check_step

pytestmark = pytest.mark.gpu

KS = [24, 32, 33, 160, 161, 200, 256, 257, 500, 1000, 1024]
LIMIT_NAMES = list(TW.CHECK_ORDER)
GROUPS = ("O1", "AT", "O2", "PAST", "O3")
NG, DEG = 8, 4                      # nodes per group (one tile), edges per node
N_TILE_NODES = NG * len(GROUPS)
N_ISO = 3
DEAD = 1.0e5


def _pick_rows(n, target, g, h, cmin, cmax):
    """n row lengths c in [cmin, cmax] with sum g(c) == target and the smallest sum h(c), or None."""
    cs = list(range(cmin, cmax + 1))
    INF = 1 << 30
    best = np.full(target + 1, INF, dtype=np.int64)
    best[0] = 0
    choice = []
    for _ in range(n):
        nb = np.full(target + 1, INF, dtype=np.int64)
        ch = np.full(target + 1, -1, dtype=np.int64)
        for c in cs:
            gc, hc = int(g(c)), int(h(c))
            if gc > target:
                continue
            cand = best[:target + 1 - gc] + hc
            better = cand < nb[gc:]
            nb[gc:][better] = cand[better]
            ch[gc:][better] = c
        best = nb
        choice.append(ch)
    if best[target] >= INF:
        return None
    out, t = [], target
    for ch in reversed(choice):
        c = int(ch[t])
        out.append(c)
        t -= int(g(c))
    return sorted(out, reverse=True)


def _deal(rows):
    """32 neighbour rows (longest first) to 8 nodes x 4 edges, round robin: node i gets rows i, i + 8, i + 16, i + 24."""
    return [[rows[i + NG * j] for j in range(DEG)] for i in range(NG)]


def _design(limit, over, K):
    """(own comps of the 8 nodes, comps of their 4 x 8 neighbour rows, dead comps) of a tile whose `limit` quantity is
    LIMITS[limit] + over, or None when that does not fit in K components."""
    L = TW.LIMITS[limit] + over
    pref = lambda c: list(range(c))
    if limit == "stage_e":           # long neighbour rows over dead components
        rows = _pick_rows(NG * DEG, L, TW.chunks, lambda c: c, 1, min(K, 40))
        if rows is None or sum(rows) > TW.LIMITS["erow"]:
            return None
        return [[0]] * NG, [[pref(c) for c in r] for r in _deal(rows)], set(range(1, K))
    if limit == "erow":              # as many entries in as few chunks as possible
        rows = _pick_rows(NG * DEG, L, lambda c: c, TW.chunks, 1, min(K, 40))
        if rows is None or int(TW.chunks(rows).sum()) > TW.LIMITS["stage_e"]:
            return None
        return [[0]] * NG, [[pref(c) for c in r] for r in _deal(rows)], set(range(1, K))
    if limit == "stage_u":           # long own rows, live
        rows = _pick_rows(NG, L, TW.chunks, lambda c: c, 1, min(K, 64))
        if rows is None:
            return None
        return [pref(c) for c in rows], [[[0]] * DEG for _ in range(NG)], set()
    if limit == "slots":             # own row 0..8 (live), the neighbours' rows cover 9..47 (dead) between them
        own = 9
        per_node = [L // NG + (1 if i < L % NG else 0) for i in range(NG)]
        if max(per_node) > K:
            return None
        nbr = []
        for span in per_node:
            rest = list(range(own, span))
            nbr.append([[0] + rest[j::DEG] for j in range(DEG)])
        return [pref(own)] * NG, nbr, set(range(own, K))
    if limit == "act":               # own row 0..7, the neighbours add live components 8..8+b-1 (active: gradient > 0)
        own = 8
        extra = L - NG * own
        per_node = [extra // NG + (1 if i < extra % NG else 0) for i in range(NG)]
        if own + max(per_node) > K:
            return None
        nbr = []
        for b in per_node:
            rest = list(range(own, own + b))
            nbr.append([[0] + rest[j::DEG] for j in range(DEG)])
        return [pref(own)] * NG, nbr, set()
    if limit == "ent":               # own row 0..6; every neighbour entry is on an active component of the node
        own = 7
        if own > K:
            return None
        rows = [own] * (NG * DEG)
        for i in range(NG * DEG * own - L):
            rows[-1 - i] -= 1
        return [pref(own)] * NG, [[pref(c) for c in r] for r in _deal(rows)], set()
    raise ValueError(limit)


def _ordinary():
    return [[0, 1]] * NG, [[[0, 2]] * DEG for _ in range(NG)], set()


def _build(specs, K, seed=0):
    """Graph, F0 and sumF of a list of groups (name, own comps per node, neighbour-row comps per node and edge, dead comps):
    the groups' nodes get ids in list order, every node its own leaves (ids after all group nodes), then N_ISO isolated
    nodes with empty rows."""
    from bigclam_apachespark_b200 import graphs as G
    n_nodes = sum(len(own) for _, own, _, _ in specs)
    n_leaves = sum(len(r) for _, _, nbr, _ in specs for r in nbr)
    n = n_nodes + n_leaves + N_ISO
    rng = np.random.default_rng(seed * 1000 + K)
    F0 = np.zeros((n, K))
    dead = set()
    us, vs = [], []
    groups = {}
    u, v = 0, n_nodes
    for name, own, nbr, dd in specs:
        dead |= dd
        groups[name] = np.arange(u, u + len(own))
        for i in range(len(own)):
            F0[u, own[i]] = 1.0
            for row in nbr[i]:
                F0[v, row] = 1.0
                us.append(u)
                vs.append(v)
                v += 1
            u += 1
    nz = F0 != 0
    F0[nz] = rng.uniform(0.3, 0.7, int(nz.sum()))
    F0[:, 0] = np.where(nz[:, 0], 0.1, 0.0)
    sumF = F0.sum(axis=0) + 1.0
    sumF[sorted(dead)] += DEAD
    rp, col = G.csr_from_undirected(n, np.array(us), np.array(vs))
    return dict(rp=rp, col=col, F0=F0, sumF=sumF, K=K, groups=groups)


def build_case(limit, over_at_past=(0, 1), K=32, seed=0):
    """Graph, F0, sumF and the node ids of the five groups; None when the construction does not fit in K."""
    designs = {"AT": _design(limit, over_at_past[0], K), "PAST": _design(limit, over_at_past[1], K)}
    if designs["AT"] is None or designs["PAST"] is None:
        return None
    case = _build([(name, *(designs.get(name) or _ordinary())) for name in GROUPS], K, seed)
    case["limit"] = limit
    case["designed"] = np.concatenate([case["groups"]["AT"], case["groups"]["PAST"]])
    _assert_design(case, over_at_past)
    return case


def _tile_of(cut, ids):
    for t, nodes in enumerate(cut["tiles"]):
        if set(nodes.tolist()) == set(ids.tolist()):
            return t
    raise AssertionError(f"nodes {ids.tolist()} are not one tile of the cut")


def _assert_design(case, over_at_past):
    """The designed tiles have the designed quantities (through the model, exhaustive search: every node with edges
    searched), and fall back exactly where they should: a construction that drifts fails here, loudly."""
    limit = case["limit"]
    cut = TW.cut(case["rp"])
    assert cut["n_hubs"] == 0 and cut["n_gen"] == 0
    for name in GROUPS:
        _tile_of(cut, case["groups"][name])
    pred = TW.predict_kernel(case["rp"], case["col"], case["F0"], case["sumF"], cut["tiles"], exhaustive=True)
    for name, over in zip(("AT", "PAST"), over_at_past):
        q, fail = pred[_tile_of(cut, case["groups"][name])]
        assert q[TW.QUANTITY[limit]] == TW.LIMITS[limit] + over, (name, limit, q)
        others = [k for k in TW.CHECK_ORDER if k != limit]
        assert all(q[TW.QUANTITY[k]] <= TW.LIMITS[k] for k in others), (name, limit, q)
        assert fail == (limit if over > 0 else None), (name, limit, q, fail)
    for name in ("O1", "O2", "O3"):
        assert pred[_tile_of(cut, case["groups"][name])][1] is None, name
    case["cut"] = cut


def _solver(case, exhaustive, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(record_accepted=True, sparse_rows=True, time_kernels=True, exhaustive_linesearch=exhaustive, **kw)
    b.set_graph(case["rp"], case["col"]).set_K(case["K"]).set_F(case["F0"], sumF=case["sumF"])
    return b


@pytest.fixture(autouse=True)
def _pinned_budget(monkeypatch):
    monkeypatch.setenv("BIGCLAM_TILE_EDGES", str(TW.MAX_EDGES))


def _first_step_counts(case, b, exhaustive, node_mask=None):
    """One step; the tile counters of its two kernels against the model; returns the step's LLH and the model's
    prediction of its first kernel."""
    rp, col, cut = case["rp"], case["col"], case["cut"]
    st = b.tile_stats()
    assert st["n_tiles"] == len(cut["tiles"]) and st["n_general_nodes"] == cut["n_gen"] and st["n_split_hubs"] == 0, st
    assert st["tiles_done"] == 0 and st["tiles_fallback"] == 0, st
    uset = None if node_mask is None else np.flatnonzero(node_mask)
    llh = b.backtrackingLineSearchs(uset)
    F1, s1 = b.F, b.sumF
    k1 = TW.predict_kernel(rp, col, case["F0"], case["sumF"], cut["tiles"], exhaustive, node_mask)
    k2 = TW.predict_kernel(rp, col, F1, s1, cut["tiles"], exhaustive, node_mask)
    st = b.tile_stats()
    d1, f1 = TW.predict_counts(k1)
    d2, f2 = TW.predict_counts(k2)
    assert (st["tiles_done"], st["tiles_fallback"]) == (d1 + d2, f1 + f2), (st, [f for _, f in k1], [f for _, f in k2])
    return llh, k1


def _three_steps(case, b, oracle, first, node_mask=None, where=""):
    rp, col, K = case["rp"], case["col"], case["K"]
    P = oracle.make_params(K)
    F, s = case["F0"], case["sumF"]
    uset = None if node_mask is None else np.flatnonzero(node_mask)
    designed = case["designed"]
    for it in range(3):
        llh = first if it == 0 else b.backtrackingLineSearchs(uset)
        r = oracle.step(rp, col, F, s, P, node_mask=node_mask)
        row_err = np.abs(b.F - r.F).max(axis=1)
        assert (row_err[designed] <= 1e-9 * max(np.abs(r.F).max(), 1e-300)).all(), f"{where} step {it}: a designed node flipped"
        # (a small graph converges within a few steps: a handful of nodes whose tiny candidates are proven ties is 3 %)
        _check_step(b, r, llh, max_flips=0, where=f"{where} step {it}", max_idx_diff=0.05, inputs=(rp, col, F, s, P))
        F, s = b.F, b.sumF


@pytest.mark.parametrize("exhaustive", [False, True], ids=["bounds", "exhaustive"])
@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("limit", LIMIT_NAMES)
def test_tile_limit_at_and_past(oracle, limit, K, exhaustive):
    """The AT tile runs on the tile path, the PAST tile falls back at the designed check; counters exact; 3 steps."""
    case = build_case(limit, K=K)
    if case is None:
        pytest.skip(f"the {limit} construction does not fit in K = {K}")
    b = _solver(case, exhaustive)
    llh, k1 = _first_step_counts(case, b, exhaustive)
    assert k1[_tile_of(case["cut"], case["groups"]["AT"])][1] is None
    assert k1[_tile_of(case["cut"], case["groups"]["PAST"])][1] == limit
    _three_steps(case, b, oracle, llh, where=f"{limit} K={K} ex={exhaustive}")
    b.close()


def test_entry_limit_with_uset(oracle):
    """The PAST tile of the TE construction overflows with every node searched and fits once the uset drops one node."""
    case = build_case("ent", over_at_past=(0, 1), K=32)
    past = case["groups"]["PAST"]
    mask = np.ones(len(case["rp"]) - 1, dtype=np.uint8)
    mask[past[0]] = 0
    full = TW.predict_kernel(case["rp"], case["col"], case["F0"], case["sumF"], case["cut"]["tiles"], True)
    part = TW.predict_kernel(case["rp"], case["col"], case["F0"], case["sumF"], case["cut"]["tiles"], True, mask)
    t = _tile_of(case["cut"], past)
    assert full[t][1] == "ent" and part[t][1] is None and part[t][0]["TE"] < full[t][0]["TE"]
    for exhaustive in (True, False):
        b = _solver(case, exhaustive)
        llh, k1 = _first_step_counts(case, b, exhaustive, node_mask=mask)
        assert k1[t][1] is None
        _three_steps(case, b, oracle, llh, node_mask=mask, where=f"uset ex={exhaustive}")
        b.close()


def test_device_loop_on_a_boundary_graph(oracle):
    """bigclam_run (the device-side loop) through the AT / PAST tiles of the active-component limit."""
    case = build_case("act", K=33)
    P = oracle.make_params(33)
    b = _solver(case, False)
    b._run(4, 0.0, 12)
    Fo, so, llho, callso, tro = oracle.run(case["rp"], case["col"], case["F0"], case["sumF"], P, variant=4, rel_tol=0.0,
                                           max_outer=12)
    assert b.last_calls == callso
    assert np.allclose(b.last_trace, tro, rtol=1e-9, atol=0.0)
    assert np.abs(b.F - Fo).max() <= 1e-9 * np.abs(Fo).max()
    st = b.tile_stats()
    assert st["tiles_fallback"] > 0 and st["tiles_done"] > 0
    b.close()


def test_rerun_is_bit_identical_on_a_boundary_graph():
    case = build_case("ent", K=161)
    out = []
    for _ in range(2):
        b = _solver(case, False)
        llhs = [b.backtrackingLineSearchs() for _ in range(3)]
        out.append((llhs, b.F.tobytes(), b.sumF.tobytes(), b.accepted().tobytes(), b.tile_stats()))
        b.close()
    assert out[0] == out[1]


def test_wide_rows_have_no_tiles(oracle):
    """K = 1025 (wide rows): the same kind of graph runs without tiles, every node on the general path."""
    case = build_case("act", K=1024)
    K = 1025
    F0 = np.zeros((len(case["rp"]) - 1, K))
    F0[:, :1024] = case["F0"]
    sumF = np.concatenate([case["sumF"], [1.0]])
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(record_accepted=True, sparse_rows=True, time_kernels=True)
    b.set_graph(case["rp"], case["col"]).set_K(K).set_F(F0, sumF=sumF)
    st = b.tile_stats()
    assert st["n_tiles"] == 0
    llh = b.backtrackingLineSearchs()
    P = oracle.make_params(K)
    r = oracle.step(case["rp"], case["col"], F0, sumF, P)
    _check_step(b, r, llh, where="wide", inputs=(case["rp"], case["col"], F0, sumF, P))
    b.close()


@pytest.mark.parametrize("exhaustive", [False, True], ids=["bounds", "exhaustive"])
@pytest.mark.parametrize("K", [24, 161, 257])
def test_degree_32_tile_next_to_degree_33_general_node(oracle, K, exhaustive):
    """The edge budget of a tile as a boundary of the cut: a degree-33 node goes to the general path, the degree-32 node
    right behind it in the processing order is a tile of one node (one lane group of 32 lanes), ordinary tiles follow."""
    ordinary = _ordinary()
    case = _build([("G33", [[0, 1]], [[[0, 2]] * 33], set()), ("T32", [[0, 1]], [[[0, 2]] * 32], set()),
                   ("O1", *ordinary), ("O2", *ordinary), ("O3", *ordinary)], K)
    g33, t32 = case["groups"]["G33"], case["groups"]["T32"]
    cut = TW.cut(case["rp"])
    assert cut["n_hubs"] == 0 and cut["n_gen"] == 1 and cut["order"][0] == g33[0] and cut["order"][1] == t32[0]
    assert _tile_of(cut, t32) == 0 and all(_tile_of(cut, case["groups"][n]) > 0 for n in ("O1", "O2", "O3"))
    case["cut"] = cut
    case["designed"] = np.concatenate([g33, t32])
    b = _solver(case, exhaustive)
    llh, k1 = _first_step_counts(case, b, exhaustive)
    assert all(f is None for _, f in k1)
    _three_steps(case, b, oracle, llh, where=f"deg 32/33 K={K} ex={exhaustive}")
    b.close()


def _dense_case(K, width, seed=0):
    """The five groups of 8 nodes of degree 4, and one node of each degree 6..32 ahead of them (a ladder: how many of its
    nodes go to the general path gives the edge budget exactly), every row (own and leaves) `width` components wide."""
    rng = np.random.default_rng(seed * 7919 + width)
    row = lambda: [0] + sorted(rng.choice(np.arange(1, K), width - 1, replace=False).tolist())
    ladder = range(6, TW.MAX_EDGES + 1)
    specs = [("LADDER", [row() for _ in ladder], [[row() for _ in range(d)] for d in ladder], set())]
    specs += [(name, [row() for _ in range(NG)], [[row() for _ in range(DEG)] for _ in range(NG)], set()) for name in GROUPS]
    case = _build(specs, K, seed)
    case["designed"] = np.concatenate([case["groups"][n] for n in ("LADDER",) + GROUPS])
    return case


@pytest.mark.parametrize("width", [20, 100])
def test_unpinned_budget_follows_retile(oracle, monkeypatch, width):
    """BIGCLAM_TILE_EDGES unset: set_F re-cuts the tiles for the rows' average size (retile).  Rows of 20 components give a
    smaller edge and node budget, rows of 100 no tiles at all; the model's restatement of retile predicts both cuts, and
    the counters of the first step follow from them."""
    monkeypatch.delenv("BIGCLAM_TILE_EDGES")
    K = 200
    case = _dense_case(K, width)
    edges, nodes = TW.retile_budget(case["rp"], case["F0"], K)
    assert (edges, nodes) != (TW.MAX_EDGES, TW.MAX_NODES)
    cut = TW.cut(case["rp"], tile_edges=edges, tile_nodes=nodes)
    assert len(cut["tiles"]) != len(TW.cut(case["rp"])["tiles"])
    if width == 20:
        assert cut["n_gen"] == TW.MAX_EDGES - edges and 2 <= nodes < TW.MAX_NODES
    if width == 100:
        assert edges == 0 and cut["tiles"] == [] and cut["n_gen"] == len(case["rp"]) - 1
    case["cut"] = cut
    b = _solver(case, True)
    llh, _ = _first_step_counts(case, b, True)
    _three_steps(case, b, oracle, llh, where=f"retile width={width} ({edges} edges, {nodes} nodes)")
    b.close()
