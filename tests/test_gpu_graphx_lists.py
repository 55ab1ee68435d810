"""The step engines on neighbour lists as GraphX gives them (collectNeighborIds(Either), bigclam4-7.scala:50, and the
product's reader at multiplicity 0): every edge line adds an entry at both ends, a repeated line another one, a self loop
line two entries u -> u, and the lists come in no particular order.  bigclam_create takes such lists as given; every
other step test builds simple, symmetric, sorted lists.

The graphs (_graph): a degree-4 random graph with a hub, run through graphx() (self loops, repeated lines, shuffled lists
and, for the "one_sided" kind, one end of some edges dropped), plus special nodes, each for a place where an entry count
is a budget or a boundary:
  * SELF_ONLY: lists of 1 to 4 self-loop entries: the node is its own only neighbour;
  * REP40: one neighbour repeated 40 times: above the 32-entry tile budget with one distinct neighbour;
  * G33 / T32: 33 and 32 entries with repeats, next to each other in the processing order: at the full tile budget of
    32 entries (rows of a few components: K = 1 and 13 here), the last node of the general path and a tile of one node
    (tests/test_gpu_tile_limits.py::test_degree_32_tile_next_to_degree_33_general_node);
  * PAIR: two nodes of 16 entries that share the tile after T32's at that budget; the first has a self loop and lists
    the other;
  * the hub repeats one neighbour at entries kSpHubSeg - 1 and kSpHubSeg, on either side of its first slice boundary
    once it is a split hub.
The special lists are one-sided: the other lists do not name the special nodes (REP40's neighbour would otherwise be a
node of 40 entries too).

Every engine case takes three steps against the oracle with _check_step (the tie proof) and the null-step prediction of
tests/test_gpu_params.py, from F0 of about 8 non-zeros per row (test_gpu_params._F0: denser rows, or lists with many repeats
of a heavy row, put every edge past x_hi, where the objective is linear in the row and whole neighbourhoods make their
Armijo decisions on rounding), and asserts which path ran: the tile counters against the cut of tests/tile_twin.py, the
line-search node counts, the replicas of a multi-GPU handle.  The tiles are cut as set_F cuts them for the rows' size
(retile; tests/tile_twin.py restates it): at K = 200 and 256 the full budget would send nearly every tile of these rows
back to the general path.  Email-Enron is the reference's own input (Bigclamv2.scala:14):
every pair listed in both directions, so under GraphX every neighbour appears twice (doubled())."""
import os

import numpy as np
import pytest

import tile_twin as TW
from conftest import random_graph
from test_gpu_links import _llh_from_edges
from test_gpu_params import DEFAULTS, _F0, _null_steps, _steps
from test_gpu_parity import RTOL_F, _check_step

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"

N = 200                  # nodes of the engine graphs
HUB = 110                # extra distinct neighbours of node 0: 100 <= entries < 2 kSpHubSeg (a split hub only when asked)
SPLIT_HUB_DEG = 100      # BIGCLAM_SPARSE_HUB_DEG of the split-hub case
SELF_ONLY = [1, 2, 3, 4]
REP40, REP40_NB = 5, 6
G33, T32 = 7, 8
PAIR = (9, 10)
SPECIAL = set(SELF_ONLY) | {REP40, G33, T32, *PAIR}


# ---------------------------------------------------------------------------------------------------------------------
# graph builders

def _lists(rp, col):
    return [[int(v) for v in col[rp[u]:rp[u + 1]]] for u in range(len(rp) - 1)]


def _csr(lists):
    rp = np.zeros(len(lists) + 1, dtype=np.int64)
    rp[1:] = np.cumsum([len(L) for L in lists])
    col = np.array([v for L in lists for v in L], dtype=np.int32)
    return rp, col


def doubled(rp, col):
    """Every entry twice, next to each other: a simple graph whose edge list names every pair in both directions (as
    Email-Enron.txt does), read by GraphX."""
    deg = np.diff(rp)
    return np.concatenate([[0], np.cumsum(2 * deg)]).astype(np.int64), np.repeat(col, 2).astype(np.int32)


def graphx(rp, col, seed, self_loop_frac=0.05, repeat_frac=0.1, shuffle=True, drop_frac=0.0):
    """The simple symmetric graph (rp, col) as edge lines read by GraphX: each edge u < v is one line, repeated once
    (repeat_frac) or twice (repeat_frac / 5) more; a self_loop_frac of the nodes get a self-loop line (two entries u -> u);
    with drop_frac, that fraction of the edge lines adds its entry at one end only (a one-sided CSR).  Lists are shuffled,
    or sorted when shuffle is False."""
    rng = np.random.default_rng(seed)
    n = len(rp) - 1
    lists = [[] for _ in range(n)]
    for u in range(n):
        for v in col[rp[u]:rp[u + 1]]:
            v = int(v)
            if v <= u:
                continue
            r = rng.random()
            mult = 1 + (r < repeat_frac) + (r < repeat_frac / 5)
            for _ in range(mult):
                d = rng.random() < drop_frac
                side = rng.random() < 0.5
                if not (d and side):
                    lists[u].append(v)
                if not (d and not side):
                    lists[v].append(u)
    for u in np.flatnonzero(rng.random(n) < self_loop_frac):
        lists[u] += [int(u), int(u)]
    for L in lists:
        if shuffle:
            rng.shuffle(L)
        else:
            L.sort()
    return _csr(lists)


def _add_special(rp, col, seed):
    """The special nodes of the module docstring on top of (rp, col); node 0 must be the hub."""
    rng = np.random.default_rng(seed + 1)
    lists = _lists(rp, col)
    n = len(lists)
    for u in range(n):
        lists[u] = [v for v in lists[u] if v not in SPECIAL]
    ordinary = np.array([u for u in range(11, n)])
    for i, u in enumerate(SELF_ONLY):
        lists[u] = [u] * (i + 1)
    lists[REP40] = [REP40_NB] * 40

    def with_repeats(distinct, extra, own=()):
        nb = [int(v) for v in rng.choice(ordinary, distinct, replace=False)]
        L = nb + [int(v) for v in rng.choice(nb, extra, replace=False)] + list(own)
        rng.shuffle(L)
        return L

    lists[G33] = with_repeats(19, 12, own=(G33, G33))
    lists[T32] = with_repeats(20, 12)
    p, q = PAIR
    lists[p] = with_repeats(10, 2, own=(p, p, q, q))
    lists[q] = with_repeats(12, 3, own=(p,))
    # the hub repeats one neighbour on either side of entry kSpHubSeg
    seg = TW._D["HubSeg"]
    h = lists[0]
    h.insert(seg, h[seg - 1])
    return _csr(lists)


_GRAPHS = {}


def _graph(kind, n=N, seed=11):
    """kind: "graphx" (symmetric lists with self loops and repeats, shuffled), "one_sided" (the same with 30 % of the
    edge lines at one end only), "sorted" (the lists of "graphx", sorted).  With the special nodes; checks that the cut puts
    them where the module docstring says."""
    key = (kind, n, seed)
    if key not in _GRAPHS:
        if kind == "sorted":
            rp, col = _graph("graphx", n, seed)
            rp, col = _csr([sorted(L) for L in _lists(rp, col)])
        else:
            rp, col = random_graph(n, 4, seed=seed, hub=HUB)
            rp, col = graphx(rp, col, seed, drop_frac=0.3 if kind == "one_sided" else 0.0)
            rp, col = _add_special(rp, col, seed)
        deg = np.diff(rp)
        assert SPLIT_HUB_DEG <= deg[0] < TW.HUB_DEG_MIN, deg[0]
        assert deg[REP40] == 40 and deg[G33] == 33 and deg[T32] == 32 and deg[PAIR[0]] == deg[PAIR[1]] == 16
        rest = np.delete(deg, [0] + sorted(SPECIAL))
        assert rest.max() < 16, rest.max()                      # PAIR are the first nodes after T32
        cut = TW.cut(rp)
        assert cut["n_hubs"] == 0 and list(cut["order"][:cut["n_gen"]]) == [0, REP40, G33]
        assert list(cut["tiles"][0]) == [T32] and list(cut["tiles"][1][:2]) == list(PAIR)
        _GRAPHS[key] = (rp, col)
    return _GRAPHS[key]


def test_builders():
    """What the graphs contain: repeats, self loops, shuffled lists, one-sided entries (and none in the symmetric kinds
    outside the special nodes)."""
    rp, col = random_graph(N, 4, seed=11, hub=HUB)
    r2, c2 = doubled(rp, col)
    assert np.array_equal(r2, 2 * rp) and np.array_equal(c2[::2], col) and np.array_equal(c2[1::2], col)
    lists = {}
    for kind in ("graphx", "one_sided", "sorted"):
        rp, col = _graph(kind)
        L = _lists(rp, col)
        lists[kind] = L
        ordinary = [u for u in range(1, N) if u not in SPECIAL]
        assert sum(u in L[u] for u in ordinary) >= 3                          # self loops, two entries each
        assert all(L[u].count(u) % 2 == 0 for u in ordinary)
        assert sum(len(L[u]) - len(set(L[u])) for u in ordinary) > 0.05 * sum(len(L[u]) for u in ordinary)
        assert max(max(L[u].count(v) for v in set(L[u]) if v != u) for u in ordinary if L[u]) <= 3
        assert all(L[u] == [u] * (i + 1) for i, u in enumerate(SELF_ONLY))
        pairs = {}
        for u in ordinary:
            for v in L[u]:
                if v != u:
                    pairs[(u, v)] = pairs.get((u, v), 0) + 1
        asym = sum(pairs.get((v, u), 0) != m for (u, v), m in pairs.items() if u and v and v not in SPECIAL)  # (hub: its
        # repeat at the slice boundary is one-sided)
        assert (asym > 0) == (kind == "one_sided"), (kind, asym)
        unsorted = sum(L[u] != sorted(L[u]) for u in range(N))
        assert (unsorted > N // 4) == (kind != "sorted"), (kind, unsorted)
    assert all(sorted(a) == sorted(b) for a, b in zip(lists["graphx"], lists["sorted"]))
    seg = TW._D["HubSeg"]
    for kind in KINDS:
        assert lists[kind][0][seg - 1] == lists[kind][0][seg]


# ---------------------------------------------------------------------------------------------------------------------
# engines

def _solver(rp, col, K, F0, sumF, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(record_accepted=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0, sumF=sumF)
    return b


def _start(oracle, kind, K, seed):
    rp, col = _graph(kind)
    F0 = _F0(len(rp) - 1, K, DEFAULTS, seed=seed)
    return rp, col, F0, oracle.colsum(F0)


def _sparse_engine(oracle, kind, K, monkeypatch, split=False):
    """Tiles + general path (K <= 1024), wide rows (K > 1024) or a split hub: the counters against the cut."""
    monkeypatch.delenv("BIGCLAM_TILE_EDGES", raising=False)                  # set_F cuts the tiles for the rows' size
    if split:
        monkeypatch.setenv("BIGCLAM_SPARSE_HUB_DEG", str(SPLIT_HUB_DEG))
    rp, col, F0, sumF = _start(oracle, kind, K, seed=K + 3)
    edges, nodes = TW.retile_budget(rp, F0, K)
    cut = TW.cut(rp, tile_edges=edges, tile_nodes=nodes, ld=K, hub_deg=SPLIT_HUB_DEG if split else None)
    if edges == TW.MAX_EDGES and K <= TW.WIDE_LD and not split:
        assert cut["order"][cut["n_gen"] - 1] == G33 and list(cut["tiles"][0]) == [T32]
    b = _solver(rp, col, K, F0, sumF, sparse_rows=True, time_kernels=True)
    st0 = b.tile_stats()
    where = f"{kind} {'split' if split else 'sparse'} K={K}"
    assert (st0["n_tiles"], st0["n_general_nodes"], st0["n_split_hubs"]) == (len(cut["tiles"]), cut["n_gen"], cut["n_hubs"]), \
        (where, st0)
    list(_steps(oracle, b, rp, col, F0, sumF, oracle.make_params(K), 3, where))
    st = b.tile_stats()
    wide = K > TW.WIDE_LD
    assert (st0["n_tiles"] > 0 and st["tiles_done"] > 0) == (not wide), (where, st0, st)
    assert st0["n_general_nodes"] >= (3 if not split else 2) and st0["n_split_hubs"] == (1 if split else 0), (where, st0)
    b.close()


KINDS = ["graphx", "one_sided"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [1, 13, 37, 200, 256, 257])
def test_tiles_and_general_path(oracle, kind, K, monkeypatch):
    _sparse_engine(oracle, kind, K, monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [1025, 2000])
def test_wide_rows(oracle, kind, K, monkeypatch):
    _sparse_engine(oracle, kind, K, monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
def test_split_hub(oracle, kind, monkeypatch):
    """The hub (100 to 191 entries) in slices of kSpHubSeg entries, one neighbour on either side of the first boundary."""
    _sparse_engine(oracle, kind, 24, monkeypatch, split=True)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [24, 200])
def test_bounds_equal_exhaustive_search(oracle, kind, K, monkeypatch):
    """The line-search bounds of the tile path and (BIGCLAM_LS_PRUNE=2) of the general path against the exhaustive search,
    bit for bit, in the large-graph regime (sumF as if the graph were 700 times larger)."""
    monkeypatch.setenv("BIGCLAM_LS_PRUNE", "2")
    rp, col, F0, sumF = _start(oracle, kind, K, seed=K + 5)
    sumF = sumF * 700.0
    P = oracle.make_params(K)
    where = f"{kind} bounds K={K}"
    bp = _solver(rp, col, K, F0, sumF, sparse_rows=True, time_kernels=True)
    bx = _solver(rp, col, K, F0, sumF, sparse_rows=True, time_kernels=True, exhaustive_linesearch=True)
    assert bp.tile_stats()["n_tiles"] > 0
    asked = searched = 0
    for r in _steps(oracle, bp, rp, col, F0, sumF, P, 3, where):
        lx = bx.backtrackingLineSearchs()
        assert np.array_equal(bp.accepted(), bx.accepted()), where
        assert bp.F.tobytes() == bx.F.tobytes() and bp.sumF.tobytes() == bx.sumF.tobytes(), where
        assert abs(lx - r.llh) <= 1e-10 * abs(r.llh), where
        st, sx = bp.ls_stats(), bx.ls_stats()
        assert sx["nodes_searched"] == sx["nodes_asked"], (where, sx)
        asked += st["nodes_asked"]
        searched += st["nodes_searched"]
    assert bp.tile_stats()["tiles_done"] > 0, where
    assert 0 < searched < asked, (where, searched, asked)
    bp.close()
    bx.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [13, 200])
def test_dense_rows(oracle, kind, K):
    rp, col, F0, sumF = _start(oracle, kind, K, seed=K + 9)
    b = _solver(rp, col, K, F0, sumF, time_kernels=True)
    list(_steps(oracle, b, rp, col, F0, sumF, oracle.make_params(K), 3, f"{kind} dense K={K}"))
    assert b.tile_stats() == dict(tiles_done=0, tiles_fallback=0, n_tiles=0, n_general_nodes=0, n_split_hubs=0)
    b.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("world", [2, 3])
def test_multi_gpu(oracle, kind, world):
    """The deal balances the ranks by list entries; the replicas must be bit-identical and match the oracle."""
    from bigclam_apachespark_b200 import _lib
    if int(_lib.load().bigclam_device_count()) < world:
        pytest.skip(f"needs {world} GPUs")
    K = 24
    rp, col, F0, sumF = _start(oracle, kind, K, seed=K + world)
    P = oracle.make_params(K)
    b = _solver(rp, col, K, F0, sumF, numGPUs=world)
    assert abs(b.loglikelihood() - oracle.llh(rp, col, F0, sumF, P)) <= 1e-10 * abs(oracle.llh(rp, col, F0, sumF, P))
    b.ls_stats()
    F, s = F0, sumF
    for it in range(3):
        where = f"{kind} world={world} step {it}"
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P)
        assert abs(llh - r.llh) <= 1e-10 * abs(r.llh), where
        assert b.last_n_updated == r.n_updated, where
        reps = [b.replica_F(q) for q in range(world)]
        for q in range(1, world):
            assert np.array_equal(reps[0], reps[q]) and np.array_equal(b.replica_sumF(0), b.replica_sumF(q)), (where, q)
        assert np.abs(reps[0] - r.F).max() <= 1e-9 * max(np.abs(r.F).max(), 1e-300), where
        assert np.allclose(b.sumF, r.sumF, rtol=1e-11, atol=1e-9), where
        F, s = reps[0], b.sumF
    assert b.ls_stats()["nodes_asked"] > 0                  # (summed over the ranks: every rank stepped its nodes)
    b.close()


# ---------------------------------------------------------------------------------------------------------------------
# Email-Enron as GraphX reads it

def test_email_enron_doubled_k50(oracle, graphs):
    """Bigclamv2.scala:14's input: 183,831 pairs, each listed in both directions, so every neighbour twice.  F0 from
    initNeighborComF on the doubled lists; five steps, the LLH, then the device loop capped at 8 calls."""
    if EMU:
        pytest.skip("Email-Enron is too large for the host emulation")
    rp1, col1, _ = graphs.load_npz_graph("email-enron")
    rp, col = doubled(rp1, col1)
    n, K = len(rp) - 1, 50
    assert n == 36692 and len(col) == 735324
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(record_accepted=True, sparse_rows=True, time_kernels=True)
    b.set_graph(rp, col)
    F0 = b.initNeighborComF(K)
    sumF0 = b.sumF
    assert set(np.unique(F0)) <= {0.0, 1.0}
    P = oracle.make_params(K)
    st0 = b.tile_stats()
    assert st0["n_tiles"] > 0 and st0["n_general_nodes"] > 0, st0
    F, s = F0, sumF0
    for it in range(5):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P, want_pre=True)
        _check_step(b, r, llh, max_flips=3, where=f"enron doubled it{it}", inputs=(rp, col, F, s, P),
                    null_steps=_null_steps(oracle, r, F, P))
        F, s = b.F, b.sumF
    assert b.tile_stats()["tiles_done"] > 0
    llh_o = oracle.llh(rp, col, F, s, P)
    assert abs(b.loglikelihood() - llh_o) <= 1e-10 * abs(llh_o)
    b.set_F(F0, sumF=sumF0)
    b._run(4, 1e-4, 8)
    Fo, so, llho, callso, tro = oracle.run(rp, col, F0, sumF0, P, variant=4, max_outer=8)
    assert b.last_calls == callso
    assert np.allclose(b.last_trace, tro, rtol=1e-9, atol=0)
    assert np.abs(b.F - Fo).max() <= RTOL_F * np.abs(Fo).max()
    # (all but about 70 rows of this F0 are zero, and a zero row without a non-zero neighbour has no candidate but
    # itself: a null step.  One step from the F0 of test_email_enron_k50_one_step, where most rows move.)
    F1 = graphs.synthetic_F0(n, K, seed=1234, density=0.05)
    s1 = oracle.colsum(F1)
    b.set_F(F1, sumF=s1)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F1, s1, P, want_pre=True)
    null = _null_steps(oracle, r, F1, P)
    assert r.n_updated - null.sum() > n // 2
    _check_step(b, r, llh, max_flips=3, where="enron doubled, synthetic F0", inputs=(rp, col, F1, s1, P), null_steps=null)
    b.close()


# ---------------------------------------------------------------------------------------------------------------------
# the device loop, list order, the LLH and uset masks

@pytest.mark.parametrize("sparse", [True, False], ids=["sparse_rows", "dense_rows"])
@pytest.mark.parametrize("variant", [4, 3, 2])
def test_run_loop_to_convergence(oracle, variant, sparse):
    """SGDFindC / MBSGD(version=3, 2) on a 400-node GraphX graph against the oracle's outer loop, as
    tests/test_gpu_parity.py::test_run_loop_matches_oracle does on a simple graph."""
    rp, col = _graph("graphx", n=400, seed=41)
    n, k = len(rp) - 1, 8
    rng = np.random.default_rng(41)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.4)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    Fo, so, llho, callso, tro = oracle.run(rp, col, F0, sumF, P, variant=variant)
    b = _solver(rp, col, k, F0, sumF, sparse_rows=sparse)
    if variant == 4:
        ret = b.SGDFindC()
    else:
        b.MBSGD(version=variant)
        ret = b.last_trace[-1]
    assert b.last_calls == callso
    assert np.allclose(b.last_trace, tro, rtol=1e-9, atol=0)
    assert abs(ret - llho) <= 1e-9 * abs(llho)
    assert np.abs(b.F - Fo).max() <= RTOL_F * np.abs(Fo).max()
    assert np.allclose(b.sumF, so, rtol=1e-8)
    b.close()


def test_list_order_does_not_matter(oracle):
    """The same lists shuffled and sorted: the same accepted indices or proven ties, rows within RTOL_TIGHT, the LLH within
    1e-10, three steps each on its own state; two fresh contexts on the shuffled lists give the same bits."""
    from oracle.oracle import StepResult
    K = 24
    rs_, cs_ = _graph("sorted")
    rh, ch = _graph("graphx")
    assert np.array_equal(rs_, rh) and not np.array_equal(cs_, ch)
    F0 = _F0(N, K, DEFAULTS, seed=71)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(K)
    bs = _solver(rs_, cs_, K, F0, sumF, sparse_rows=True)
    bh = _solver(rh, ch, K, F0, sumF, sparse_rows=True)
    F, s = F0, sumF
    for it, r in enumerate(_steps(oracle, bs, rs_, cs_, F0, sumF, P, 3, "sorted")):
        llh_h = bh.backtrackingLineSearchs()
        rs = StepResult(bs.F, bs.sumF, bs.loglikelihood(), bs.last_n_updated,
                        bs.accepted(), None, None, None)
        _check_step(bh, rs, llh_h, max_flips=1, where=f"shuffled vs sorted step {it}", inputs=(rs_, cs_, F, s, P))
        F, s = bs.F, bs.sumF
    bs.close()
    bh.close()
    out = []
    for _ in range(2):
        b = _solver(rh, ch, K, F0, sumF, sparse_rows=True)
        llh = b._run(4, 0.0, 7)
        out.append((llh, b.last_trace.tobytes(), b.F.tobytes(), b.sumF.tobytes()))
        b.close()
    assert out[0] == out[1]


@pytest.mark.parametrize("sparse", [True, False], ids=["sparse_rows", "dense_rows"])
def test_llh_from_entries_with_multiplicity(oracle, sparse):
    """sum_u [ sum_{v in N(u)} (log p_uv + x_uv) - F_u . sumF + x_uu ] over the list entries, repeats and self loops
    each at their multiplicity, is loglikelihood() (tests/test_gpu_links.py on simple graphs)."""
    K = 37
    rp, col, F0, sumF = _start(oracle, "one_sided", K, seed=37)
    b = _solver(rp, col, K, F0, sumF, sparse_rows=sparse)
    for _ in range(3):
        b.backtrackingLineSearchs()
    llh = b.loglikelihood()
    assert abs(_llh_from_edges(b, rp, col) - llh) <= 1e-10 * abs(llh)
    llh_o = oracle.llh(rp, col, b.F, b.sumF, oracle.make_params(K))
    assert abs(llh - llh_o) <= 1e-10 * abs(llh_o)
    b.close()


@pytest.mark.parametrize("sparse", [True, False], ids=["sparse_rows", "dense_rows"])
def test_uset_mask(oracle, sparse):
    """Nodes outside the uset keep their rows bit for bit, among them self-loop nodes (a node that is its own only
    neighbour, and a tile node with a self loop); self-loop nodes inside the uset step as the oracle says."""
    K = 13
    rp, col, F0, sumF = _start(oracle, "graphx", K, seed=13)
    rng = np.random.default_rng(13)
    P = oracle.make_params(K)
    b = _solver(rp, col, K, F0, sumF, sparse_rows=sparse)
    F, s = F0, sumF
    for it in range(2):
        mask = (rng.random(N) < 0.5).astype(np.uint8)
        out, into = (SELF_ONLY[1], PAIR[0]), (SELF_ONLY[3], G33)
        if it == 1:
            out, into = into, out
        mask[list(out)] = 0
        mask[list(into)] = 1
        llh = b.backtrackingLineSearchs(uset=np.flatnonzero(mask))
        r = oracle.step(rp, col, F, s, P, node_mask=mask)
        _check_step(b, r, llh, where=f"uset sparse={sparse} step {it}", inputs=(rp, col, F, s, P))
        Fn = b.F
        assert np.array_equal(Fn[mask == 0], F[mask == 0])
        F, s = Fn, b.sumF
    b.close()
