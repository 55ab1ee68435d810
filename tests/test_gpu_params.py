"""The step away from the script's parameter values (bigclam4-7.scala:22-26,39-43): MaxInter, alpha, beta, MIN_P_/MAX_P_,
MIN_F_ and MAX_F_ as the C API accepts them, on every engine that takes them, step after step against the oracle with the
GPU on its own state; the rejected values; fold-in and edge_probability at non-default values.

Every engine case asserts which path ran (tile counters, split hubs, the bounds' node counts), so that none can pass on
a fallback.  Tolerances are those of tests/test_gpu_parity.py (_check_step: TIE_TOL and the tie proof); the one thing
added is the prediction of where the accepted index may differ at any rate: nodes whose every candidate is their own row
(see _check_step's `null_steps`).  At MIN_P_ = 0.05 / MAX_P_ = 0.95 those are common: a zero row has x = 0 on every
edge, p is clamped at MAX_P_, and its gradient sum_v F_v / (1 - MAX_P_) - sumF is negative in every component once
1 / (1 - MAX_P_) is only 20, so every candidate is the zero row again."""
import os

import numpy as np
import pytest

from conftest import random_graph
from test_gpu_parity import _check_step

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"

DEFAULTS = dict(alpha=0.05, beta=0.1, MaxInter=15, MIN_P_=0.0001, MAX_P_=0.9999, MIN_F_=0.0, MAX_F_=1000.0)

# name -> the values away from the defaults; the comment names the branch each set is for
SETS = {
    "mi0": dict(MaxInter=0),                    # one candidate (s = 1)
    "mi3": dict(MaxInter=3),                    # a group of 4 candidates inside the 16-lane scan
    "mi15": dict(MaxInter=15),                  # nsteps = 16: the last count with tiles, split hubs and bound_mask
    "mi16": dict(MaxInter=16),                  # nsteps = 17: no tiles, no split hubs, a second group of 16 candidates
    "mi17": dict(MaxInter=17),                  # the grouped scan (tg += 16), two groups
    "mi40": dict(MaxInter=40, beta=0.5),        # the grouped scan, three groups (s down to 1e-12)
    "mi63": dict(MaxInter=63, beta=0.6),        # the largest count kMaxSteps allows, four groups
    "beta05": dict(beta=0.5, MaxInter=40),      # slow decay: the accepted index moves deep into the candidates
    "beta09": dict(beta=0.9, MaxInter=63),      # slower still: many passing candidates, the first one wins
    "beta1": dict(beta=1.0, MaxInter=20),       # every step is 1.0: equal candidates, accept at 0 or nowhere
    "alpha0": dict(alpha=0.0),                  # ls_prune off (the bounds need alpha > 0)
    "alpha1e-6": dict(alpha=1e-6),              # bounds on, cannot_pass with an almost flat Armijo line
    "alpha03": dict(alpha=0.3),                 # cannot_pass with a steep Armijo line
    "alpha05": dict(alpha=0.5),                 # most nodes fail every candidate
    "p05": dict(MIN_P_=0.05, MAX_P_=0.95),      # many edges clamped on both sides (x_lo = 0.051, x_hi = 3.0)
    "p1e-12": dict(MIN_P_=1e-12, MAX_P_=1 - 1e-12),   # EdgeConst's 1e-12 widening next to the clamps; pr_kinv = 1e12
    "p_asym": dict(MIN_P_=1e-6, MAX_P_=0.5),    # asymmetric clamps: x_lo = log 2, pr_kinv = 2
    "maxf05": dict(MAX_F_=0.5),                 # the upper clamp binds on many rows: kap0 and G1 from MAX_F_
    "maxf2": dict(MAX_F_=2.0),                  # the same with fewer rows at the clamp (need_hi decided per node)
}
SETS_MIN_F = {                                  # dense rows only (sparse rows store no MIN_F_)
    "minf_eq_maxf": dict(MIN_F_=0.25, MAX_F_=0.25),   # every candidate is the row itself
    "minf0.01_maxf2": dict(MIN_F_=0.01, MAX_F_=2.0),  # both clamps of dense_linesearch and the write-back
}


def _params(kw):
    return dict(DEFAULTS, **kw)


def _oracle_params(oracle, K, v):
    return oracle.make_params(K, alpha=v["alpha"], beta=v["beta"], max_inter=v["MaxInter"], min_p=v["MIN_P_"],
                              max_p=v["MAX_P_"], min_f=v["MIN_F_"], max_f=v["MAX_F_"])


def _solver(v, rp, col, K, F0, sumF, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(alpha=v["alpha"], beta=v["beta"], MaxInter=v["MaxInter"], **kw)
    b.MIN_P_, b.MAX_P_, b.MIN_F_, b.MAX_F_ = v["MIN_P_"], v["MAX_P_"], v["MIN_F_"], v["MAX_F_"]
    b.set_graph(rp, col).set_K(K).set_F(F0, sumF=sumF)
    return b


def _F0(n, K, v, seed):
    """About 8 non-zeros per row (at least 5 % of K up to K = 256), values up to 3, then inside [MIN_F_, MAX_F_]: at
    MAX_F_ <= 2 many components start at the upper clamp, at MIN_F_ > 0 every zero is lifted to it.  (Rows with 50 and more
    such values would put every edge past x_hi, where the objective is linear in the row and the Armijo decisions of
    whole neighbourhoods sit at rounding level.)"""
    rng = np.random.default_rng(seed)
    F0 = 3.0 * rng.random((n, K)) * (rng.random((n, K)) < min(1.0, 8.0 / K + (0.05 if K <= 256 else 0.0)))
    return np.clip(F0, v["MIN_F_"], v["MAX_F_"])


def _null_steps(oracle, r, F, P):
    """Nodes whose every candidate row clamp(F_u + s_j g_u, MIN_F_, MAX_F_) is F_u itself (r: oracle step with want_pre)."""
    null = np.ones(len(F), dtype=bool)
    for s in np.unique(oracle.step_sizes(P.beta, P.max_inter)):
        null &= (np.clip(F + s * r.grad, P.min_f, P.max_f) == F).all(axis=1)
    return null


def _steps(oracle, b, rp, col, F, sumF, P, steps, where):
    """`steps` steps of b on its own state, each against one oracle step from the same F and sumF.  At alpha = 0 the
    Armijo line is flat: a candidate passes when its LLH does not drop, so a node at a minimum along its gradient decides
    its smallest candidates on the last bits of llh_u either way (the tie proof checks each one), and its row moves by
    s g with s down to beta^MaxInter: such rows are flips of up to 1e-8 rather than the odd one."""
    max_flips = 1 if P.alpha > 0 else 10
    for it in range(steps):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, sumF, P, want_pre=True)
        _check_step(b, r, llh, max_flips=max_flips, where=f"{where} step {it}", inputs=(rp, col, F, sumF, P),
                    null_steps=_null_steps(oracle, r, F, P))
        F, sumF = b.F, b.sumF
        yield r


def _graph(n=300, hub=120):
    """Degree-6 random graph with a hub: the hub is a block-shared node of the dense engine (degree >= 48), a node of the
    general path on sparse rows (above the 32-edge tile budget) and a split hub once BIGCLAM_SPARSE_HUB_DEG <= its
    degree; the other nodes go into tiles."""
    return random_graph(n, 6, seed=n + hub, hub=hub)


# ---------------------------------------------------------------------------------------------------------------------
# engines

ENGINES = ["dense", "sparse", "wide", "bounds", "split_hub", "multi2"]


def _run_engine(oracle, engine, name, kw, monkeypatch):
    v = _params(kw)
    nsteps = v["MaxInter"] + 1
    rp, col = _graph()
    K = {"dense": 13, "sparse": 13, "wide": 1025, "bounds": 24, "split_hub": 24, "multi2": 24}[engine]
    F0 = _F0(len(rp) - 1, K, v, seed=K + len(name))
    sumF = oracle.colsum(F0)
    P = _oracle_params(oracle, K, v)
    where = f"{name} {engine} K={K}"
    if engine == "dense":
        b = _solver(v, rp, col, K, F0, sumF, record_accepted=True)
        rs = list(_steps(oracle, b, rp, col, F0, sumF, P, 3, where))
    elif engine in ("sparse", "wide", "split_hub"):
        if engine == "split_hub":
            monkeypatch.setenv("BIGCLAM_SPARSE_HUB_DEG", "100")
        b = _solver(v, rp, col, K, F0, sumF, record_accepted=True, sparse_rows=True, time_kernels=True)
        st0 = b.tile_stats()
        rs = list(_steps(oracle, b, rp, col, F0, sumF, P, 3, where))
        st = b.tile_stats()
        tiles = nsteps <= 16 and engine != "wide"
        assert (st0["n_tiles"] > 0) == tiles and (st["tiles_done"] > 0) == tiles, (where, st0, st)
        assert st0["n_general_nodes"] >= (1 if engine != "split_hub" or nsteps > 16 else 0), (where, st0)
        assert st0["n_split_hubs"] == (1 if engine == "split_hub" and nsteps <= 16 else 0), (where, st0)
    elif engine == "bounds":
        # the bounds of the tile path and (BIGCLAM_LS_PRUNE=2) of the general path against the exhaustive search, bit for
        # bit; sumF as if the graph were 700 times larger, the regime where the bounds exclude most nodes
        monkeypatch.setenv("BIGCLAM_LS_PRUNE", "2")
        sumF = sumF * 700.0
        bp = _solver(v, rp, col, K, F0, sumF, record_accepted=True, sparse_rows=True, time_kernels=True)
        bx = _solver(v, rp, col, K, F0, sumF, record_accepted=True, sparse_rows=True, time_kernels=True,
                     exhaustive_linesearch=True)
        asked = searched = 0
        rs = []
        for r in _steps(oracle, bp, rp, col, F0, sumF, P, 3, where):
            lx = bx.backtrackingLineSearchs()
            assert np.array_equal(bp.accepted(), bx.accepted()), where
            assert bp.F.tobytes() == bx.F.tobytes() and bp.sumF.tobytes() == bx.sumF.tobytes(), where
            assert abs(lx - r.llh) <= 1e-10 * abs(r.llh), where
            st, sx = bp.ls_stats(), bx.ls_stats()
            assert sx["nodes_searched"] == sx["nodes_asked"], (where, sx)
            asked += st["nodes_asked"]
            searched += st["nodes_searched"]
            rs.append(r)
        bx.close()
        b = bp
        assert asked > 0, where
        if nsteps <= 16:
            # the bounds need alpha > 0 (and MIN_F_ == 0): at alpha = 0 every node that asks is searched
            assert (searched < asked) == (v["alpha"] > 0), (where, searched, asked)
    else:
        from bigclam_apachespark_b200 import _lib
        if int(_lib.load().bigclam_device_count()) < 2:
            pytest.skip("needs 2 GPUs")
        b = _solver(v, rp, col, K, F0, sumF, numGPUs=2)
        F, s = F0, sumF
        rs = []
        for it in range(3):
            llh = b.backtrackingLineSearchs()
            r = oracle.step(rp, col, F, s, P)
            assert abs(llh - r.llh) <= 1e-10 * abs(r.llh), (where, it)
            reps = [b.replica_F(q) for q in range(2)]
            assert np.array_equal(reps[0], reps[1]) and np.array_equal(b.replica_sumF(0), b.replica_sumF(1)), (where, it)
            assert np.abs(reps[0] - r.F).max() <= 1e-9 * max(np.abs(r.F).max(), 1e-300), (where, it)
            assert np.allclose(b.sumF, r.sumF, rtol=1e-11, atol=1e-9), (where, it)
            F, s = reps[0], b.sumF
            rs.append(r)
    b.close()
    return rs


# Wide rows at MaxInter 16 and 17 with beta 0.1: the 17th and 18th candidates (s = 1e-16, 1e-17) move a row by less than
# the rounding of its LLH sums, so every node that fails the first 16 decides them on rounding (each one passes the tie
# proof), and the wide engine's order of summation is the farthest from the oracle's: 3 to 10 % of the nodes.  mi40 and
# mi63 take the grouped scan of wide rows with candidates above that level.
CASES = [(name, engine) for name in SETS for engine in ENGINES if not (engine == "wide" and name in ("mi16", "mi17"))]


@pytest.mark.parametrize("name,engine", CASES)
def test_engine_at_parameter_set(oracle, name, engine, monkeypatch):
    rs = _run_engine(oracle, engine, name, SETS[name], monkeypatch)
    if name == "beta1":
        assert set(np.unique(rs[0].accepted)) <= {-1, 0}


@pytest.mark.parametrize("name", list(SETS_MIN_F))
def test_dense_at_min_f_set(oracle, name, monkeypatch):
    _run_engine(oracle, "dense", name, SETS_MIN_F[name], monkeypatch)


@pytest.mark.parametrize("K", [1, 5, 10, 11, 12, 13, 63, 65, 200, 1023])
@pytest.mark.parametrize("min_f", [0.001, 0.01])
def test_dense_min_f_keeps_the_padding_at_zero(oracle, min_f, K):
    """Dense rows are ld = (K + 3) & ~3 wide.  With MIN_F_ > 0 the candidates and the new row must leave the padding
    columns K .. ld - 1 at 0: lifted to MIN_F_ they enter the candidate LLH, the row and sumF, and every later dot product.
    A hub of 420 edges takes the block-shared path of the dense engine (split over blocks, K <= 256)."""
    v = _params(dict(MIN_F_=min_f))
    n, hub = (150, 100) if EMU else (500, 420)          # (the host emulation runs the split hub's blocks one after another)
    rp, col = random_graph(n, 6, seed=K, hub=hub)
    F0 = _F0(n, K, v, seed=K)
    sumF = oracle.colsum(F0)
    P = _oracle_params(oracle, K, v)
    b = _solver(v, rp, col, K, F0, sumF, record_accepted=True)
    rs = list(_steps(oracle, b, rp, col, F0, sumF, P, 3, f"min_f={min_f} K={K}"))
    assert rs[0].n_updated > 0
    assert b.F.min() >= min_f
    b.close()


# ---------------------------------------------------------------------------------------------------------------------
# rejected values

def _err(e):
    return str(e.value)


@pytest.mark.parametrize("attr,value,code,msg", [
    ("MaxInter", -1, "EUNSUPPORTED", "max_inter must be in [0,63]"),
    ("MaxInter", 64, "EUNSUPPORTED", "max_inter must be in [0,63]"),
    ("MIN_P_", 0.0, "EINVAL", "need 0 < min_p < max_p < 1"),
    ("MIN_P_", -1e-4, "EINVAL", "need 0 < min_p < max_p < 1"),
    ("MIN_P_", 0.9999, "EINVAL", "need 0 < min_p < max_p < 1"),
    ("MIN_P_", 0.99995, "EINVAL", "need 0 < min_p < max_p < 1"),
    ("MAX_P_", 1.0, "EINVAL", "need 0 < min_p < max_p < 1"),
    ("MIN_F_", 1000.5, "EINVAL", "min_f > max_f"),
    ("MAX_F_", -1.0, "EINVAL", "min_f > max_f"),
])
@pytest.mark.parametrize("sparse", [False, True])
def test_rejected_values_leave_the_other_context_usable(oracle, attr, value, code, msg, sparse):
    """A rejected create returns its code and message, and a context that exists already keeps its F and steps on as
    before; the same handle then creates a context once the value is valid again."""
    from bigclam_apachespark_b200 import BigClam, _lib
    rp, col = _graph(120, 40)
    K = 11
    v = _params({})
    F0 = _F0(len(rp) - 1, K, v, seed=3)
    sumF = oracle.colsum(F0)
    good = _solver(v, rp, col, K, F0, sumF, record_accepted=True, sparse_rows=sparse)
    bad = BigClam(record_accepted=True, sparse_rows=sparse)
    setattr(bad, attr, value)
    bad.set_graph(rp, col)
    with pytest.raises(_lib.BigclamError) as e:
        bad.set_K(K)
    assert e.value.code == getattr(_lib, code) and msg in _err(e), _err(e)
    assert good.F.tobytes() == F0.tobytes() and good.sumF.tobytes() == sumF.tobytes()
    P = _oracle_params(oracle, K, v)
    list(_steps(oracle, good, rp, col, F0, sumF, P, 1, f"after {attr}={value}"))
    setattr(bad, attr, DEFAULTS[attr])
    bad.set_K(K).set_F(F0, sumF=sumF)
    list(_steps(oracle, bad, rp, col, F0, sumF, P, 1, f"{attr} valid again"))
    good.close()
    bad.close()


def test_min_f_needs_dense_rows_one_gpu_and_no_fold_in(oracle):
    """MIN_F_ != 0: sparse rows and a multi-GPU handle (sparse rows on every rank) refuse it at create; fold-in (both calls)
    refuses it on a dense context, which keeps its F and sumF and steps on against the oracle."""
    from bigclam_apachespark_b200 import BigClam, _lib
    rp, col = _graph(120, 40)
    n, K = len(rp) - 1, 10
    v = _params(dict(MIN_F_=0.01))
    F0 = _F0(n, K, v, seed=5)
    sumF = oracle.colsum(F0)
    for kw in (dict(sparse_rows=True), dict(numGPUs=2, devices=[0, 0])):
        b = BigClam(**kw)
        b.MIN_F_ = 0.01
        b.set_graph(rp, col)
        with pytest.raises(_lib.BigclamError) as e:
            b.set_K(K)
        assert e.value.code == _lib.EUNSUPPORTED and "BIGCLAM_F_SPARSE_ROWS needs min_f == 0" in _err(e), _err(e)
        b.close()
    b = _solver(v, rp, col, K, F0, sumF, record_accepted=True)
    lib = _lib.load()
    qrp = np.array([0, 2, 3], dtype=np.int64)
    qcol = np.array([0, 1, 5], dtype=np.int32)
    with pytest.raises(_lib.BigclamError) as e:
        b.fold_in(qrp, qcol)
    assert e.value.code == _lib.EUNSUPPORTED and "needs min_f == 0 (min_f = 0.01)" in _err(e), _err(e)
    ip, ix, vl = np.zeros(3, dtype=np.int64), np.zeros(3 * K, dtype=np.int32), np.zeros(3 * K)
    rc = lib.bigclam_fold_in(b._ctx, 2, qrp.ctypes.data, qcol.ctypes.data, 10, 1e-4, ip.ctypes.data, ix.ctypes.data,
                             vl.ctypes.data, None, None)
    assert rc == _lib.EUNSUPPORTED and b"needs min_f == 0" in lib.bigclam_last_error(b._ctx)
    assert b.F.tobytes() == F0.tobytes() and b.sumF.tobytes() == sumF.tobytes()
    list(_steps(oracle, b, rp, col, F0, sumF, _oracle_params(oracle, K, v), 2, "after the fold-in refusal"))
    b.close()


# ---------------------------------------------------------------------------------------------------------------------
# fold-in and the pair queries

@pytest.mark.parametrize("sparse", [True, False])
@pytest.mark.parametrize("name", ["mi3", "mi17", "alpha03", "beta05", "maxf05", "p05"])
def test_fold_in_at_parameter_set(oracle, name, sparse):
    """Fold-in runs the step's own line search: at non-default values against the loop of oracle steps."""
    from test_gpu_fold_in import _check_against_oracle, _queries
    v = _params(SETS[name])
    rp, col = random_graph(120 if EMU else 300, 6, seed=41)
    n, K = len(rp) - 1, 37
    F0 = _F0(n, K, v, seed=41)
    b = _solver(v, rp, col, K, F0, None, sparse_rows=sparse)
    for _ in range(2):
        b.backtrackingLineSearchs()
    qrp, qcol = _queries(n, b.F, seed=41, count=8 if EMU else 30)
    _check_against_oracle(b, rp, col, qrp, qcol, max_iter=40, rel_tol=1e-4, params=_oracle_params(oracle, K, v))
    b.close()


@pytest.mark.parametrize("sparse", [True, False])
@pytest.mark.parametrize("name", ["p05", "p1e-12", "p_asym"])
def test_edge_probability_at_clamp_set(name, sparse):
    from links_twin import Twin
    from test_gpu_links import _F0 as links_F0, _bits, _pairs
    v = _params(SETS[name])
    n, K = 300, 37
    rp, col = random_graph(n, 6, seed=K)
    F0 = links_F0(n, K, seed=K)
    F0[5] = 0.0
    F0[5, 0] = np.sqrt(-np.log(v["MAX_P_"]))                        # x_55 right at x_lo = -log(MAX_P_)
    b = _solver(v, rp, col, K, F0, None, sparse_rows=sparse)
    u, v_ = _pairs(n, seed=K)
    x, p = b.edge_probability(u, v_)
    tw = Twin(*b.F_csr(), b.K, b.MIN_P_, b.MAX_P_)
    assert np.array_equal(_bits(x), _bits(tw.x(u, v_)))
    assert np.abs(p - tw.p(x)).max() <= 1e-15
    assert p[-n + 3] == 1.0 - b.MIN_P_ and p[-n + 0] == 1.0 - b.MAX_P_
    assert (p >= 1.0 - b.MAX_P_).all() and (p <= 1.0 - b.MIN_P_).all()
    b.close()
