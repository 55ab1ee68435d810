"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle.

Tolerance (BASELINE.json north_star): F within 1e-4 relative, identical top-community
assignment.  Everything is fp64 on both sides, so the observed agreement is ~1e-13; the Armijo
test is a discontinuity, so a node whose candidate sits within rounding noise of the threshold may
legitimately pick a different step (the reference itself has that freedom: Spark's reduction order
is unspecified, SURVEY T9).  Tests therefore compare rows tightly where the accepted step index
agrees and bound the number of disagreements.
"""
import numpy as np
import pytest

from conftest import random_graph, tiny_graph

pytestmark = pytest.mark.gpu

RTOL_F = 1e-4          # the contract
RTOL_TIGHT = 1e-9      # what fp64 on both sides should give


def _solver(rp, col, K, F0, sumF=None, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(record_accepted=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0, sumF=sumF)
    return b


TIE_TOL = 1e-9          # a differing Armijo decision must be a tie: |llh'(s) - rhs| <= TIE_TOL * max(|llh_u|, 1)


def _check_step(b, r, llh, max_flips=0, where="", max_idx_diff=0.02, inputs=None, null_steps=None):
    """Rows must agree tightly; a "flip" is a row that does not (an Armijo decision that went the other way).
    Every node whose accepted index differs from the oracle's — flipped row or not — must be a GENUINE TIE
    (SURVEY 8c property iv): at the first candidate where the two decision sequences part, the oracle's own
    Armijo margin llh'(s) - (llh_u + alpha s |g|^2) is at rounding level, and the step the GPU accepted passes
    the oracle's test up to that noise.  `inputs` = (rowptr, col, F_in, sumF_in, params) of the step.
    `null_steps`: mask of the nodes whose every candidate is their own row (each component pinned at a clamp).  Their
    candidate LLH is llh_u itself, so they accept the first step whose alpha s |g|^2 vanishes when added to llh_u: a
    question of the last bit of |g|^2, at any rate.  Their rows must stay as they are; they are left out of the
    max_idx_diff count."""
    F = b.F
    acc = b.accepted()
    scale = max(np.abs(r.F).max(), 1e-300)
    row_err = np.abs(F - r.F).max(axis=1)
    flipped = row_err > RTOL_TIGHT * scale
    flips = int(flipped.sum())
    assert flips <= max_flips, f"{where}: {flips} rows differ (max err {row_err.max():.3e}, scale {scale:.3e})"
    idx_diff = acc != r.accepted
    assert not (flipped & ~idx_diff).any(), f"{where}: rows differ although the accepted step is the same"
    if idx_diff.any():
        assert inputs is not None, f"{where}: accepted indices differ and no inputs were given to prove the ties"
        from oracle import oracle as O
        rp_, col_, F_in, sumF_in, params = inputs
        nodes = np.nonzero(idx_diff)[0]
        margins, llh_u = O.armijo_margins(rp_, col_, np.ascontiguousarray(F_in), sumF_in, params, nodes)
        nsteps = margins.shape[1]
        for i, u in enumerate(nodes):
            a, o = int(acc[u]), int(r.accepted[u])
            a1, o1 = (a if a >= 0 else nsteps), (o if o >= 0 else nsteps)
            j0 = min(a1, o1)
            tol = TIE_TOL * max(abs(llh_u[i]), 1.0)
            assert abs(margins[i, j0]) <= tol, (f"{where}: node {u} gpu idx {a} oracle idx {o}: margin "
                                                f"{margins[i, j0]:.3e} at candidate {j0} is not a tie (tol {tol:.1e})")
            if a >= 0:
                assert margins[i, a] >= -tol, f"{where}: node {u}: accepted candidate {a} fails the oracle's Armijo test"
    counted = idx_diff
    if null_steps is not None:
        assert np.array_equal(F[null_steps], inputs[2][null_steps]), f"{where}: a row without a candidate of its own changed"
        counted = idx_diff & ~null_steps
    assert counted.mean() <= max_idx_diff, where
    if flips == 0:
        assert np.allclose(b.sumF, r.sumF, rtol=1e-11, atol=1e-9), where
        assert abs(llh - r.llh) <= 1e-10 * abs(r.llh), where
        # the top community: one of the oracle's largest components (rows at MAX_F_ have several equal ones); rows below the
        # row tolerance have none (a tie at a tiny step may leave a row of 1e-28 on one side)
        nz = r.F.max(axis=1) > RTOL_TIGHT * scale
        top = r.F[np.arange(len(F)), F.argmax(axis=1)]
        assert (top[nz] >= r.F.max(axis=1)[nz] - RTOL_TIGHT * scale).all(), where
        if not idx_diff.any():
            assert b.last_n_updated == r.n_updated
    else:
        assert row_err[~flipped].max() <= RTOL_TIGHT * scale
    assert (F >= 0).all() and (F <= 1000).all()
    return flips


@pytest.mark.parametrize("k", [1, 2, 3, 5, 10, 31, 64, 65, 100, 200, 257, 500, 1000])
def test_single_step_all_k(oracle, k):
    """Every lane-ownership shape (C2 = 1..16 double2 chunks), odd K, K not a multiple of 4."""
    n = 400 if k <= 257 else 150
    rp, col = random_graph(n, 6, seed=k, hub=60)
    rng = np.random.default_rng(k)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < min(1.0, 8.0 / k + 0.05))
    sumF = oracle.colsum(F0)
    b = _solver(rp, col, k, F0, sumF)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, sumF, oracle.make_params(k))
    _check_step(b, r, llh, where=f"k={k}", inputs=(rp, col, F0, sumF, oracle.make_params(k)))
    b.close()


def test_dense_rows_take_dense_path(oracle):
    """More than 64 active components per row -> lane-owned dense line search."""
    n, k = 300, 200
    rp, col = random_graph(n, 5, seed=77, hub=40)
    rng = np.random.default_rng(77)
    F0 = rng.random((n, k)) * 0.2
    F0[::3] *= (rng.random((n // 3, k)) < 0.1)         # a third of the rows stay sparse
    sumF = oracle.colsum(F0)
    b = _solver(rp, col, k, F0, sumF)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, sumF, oracle.make_params(k))
    _check_step(b, r, llh, where="dense", inputs=(rp, col, F0, sumF, oracle.make_params(k)))
    b.close()


def test_golden_tiny_and_isolated_nodes(oracle, golden, graphs):
    rp, col = tiny_graph(graphs)
    F = golden["tiny_F0"]
    b = _solver(rp, col, 5, F, oracle.colsum(F))
    for it in range(3):
        llh = b.backtrackingLineSearchs()
        assert abs(llh - golden[f"tiny_llh_{it}"]) <= 1e-10 * abs(golden[f"tiny_llh_{it}"])
        acc, gold = b.accepted(), golden[f"tiny_accepted_{it}"]
        diff = acc != gold
        assert (((acc[diff] < 0) | (acc[diff] >= 12)) & ((gold[diff] < 0) | (gold[diff] >= 12))).all()
        assert np.allclose(b.F, golden[f"tiny_F_{it}"], rtol=RTOL_TIGHT, atol=1e-12)
        assert np.array_equal(b.F[10:], F[10:])          # empty neighbour lists: rows never change
    b.close()


def test_facebook_k10_multi_step_against_golden_and_oracle(oracle, golden, graphs):
    rp, col, _ = graphs.load_npz_graph("facebook_combined")
    n, K = len(rp) - 1, 10
    F = graphs.synthetic_F0(n, K, seed=1234, density=0.3)
    sumF = oracle.colsum(F)
    b = _solver(rp, col, K, F, sumF)
    P = oracle.make_params(K)
    total_flips = 0
    for it in range(6):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, sumF, P)
        total_flips += _check_step(b, r, llh, max_flips=2, where=f"facebook it{it}", inputs=(rp, col, F, sumF, P))
        if it < 3 and total_flips == 0:
            assert abs(llh - golden[f"facebook_llh_{it}"]) <= 1e-10 * abs(golden[f"facebook_llh_{it}"])
            assert (b.accepted() == golden[f"facebook_accepted_{it}"]).mean() > 0.99
        # continue from the GPU state so that errors would compound if there were any
        F, sumF = b.F, b.sumF
    b.close()


def test_uset_mask(oracle):
    n, k = 500, 12
    rp, col = random_graph(n, 5, seed=5)
    rng = np.random.default_rng(5)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.4)
    sumF = oracle.colsum(F0)
    uset = rng.choice(n, size=123, replace=False)
    mask = np.zeros(n, dtype=np.uint8)
    mask[uset] = 1
    b = _solver(rp, col, k, F0, sumF)
    llh = b.backtrackingLineSearchs(uset=uset)
    r = oracle.step(rp, col, F0, sumF, oracle.make_params(k), node_mask=mask)
    _check_step(b, r, llh, where="mask", inputs=(rp, col, F0, sumF, oracle.make_params(k)))
    assert np.array_equal(b.F[mask == 0], F0[mask == 0])
    b.close()


def test_multiplicity_kept_and_clamp_at_max_f(oracle):
    """Doubled neighbour lists (Email-Enron as GraphX reads it, SURVEY T1) drive F to MAX_F_."""
    n, k = 200, 6
    rp, col = random_graph(n, 4, seed=9)
    # duplicate every neighbour entry
    deg = np.diff(rp)
    rp2 = np.concatenate([[0], np.cumsum(2 * deg)]).astype(np.int64)
    col2 = np.repeat(col, 2).astype(np.int32)
    rng = np.random.default_rng(9)
    F = rng.random((n, k)) * 5
    sumF = oracle.colsum(F)
    b = _solver(rp2, col2, k, F, sumF)
    P = oracle.make_params(k)
    hit_max = False
    for it in range(8):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp2, col2, F, sumF, P)
        _check_step(b, r, llh, max_flips=1, where=f"dup it{it}", max_idx_diff=0.25, inputs=(rp2, col2, F, sumF, P))   # rows pinned at MAX_F_: nf == fu, pure noise decisions
        F, sumF = b.F, b.sumF
        hit_max |= bool((F == 1000.0).any())
    b.close()


def test_sumF_injection_and_drift(oracle):
    """set_sumF injects a sumF that differs from colsum(F) (the reference never recomputes it, T6)."""
    n, k = 300, 9
    rp, col = random_graph(n, 5, seed=21)
    rng = np.random.default_rng(21)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.5)
    sumF = oracle.colsum(F0) * (1 + 1e-3 * rng.standard_normal(k))
    b = _solver(rp, col, k, F0, sumF)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, sumF, oracle.make_params(k))
    _check_step(b, r, llh, where="drift", inputs=(rp, col, F0, sumF, oracle.make_params(k)))
    # and without injection the library's own column sums match the exact ones
    b2 = _solver(rp, col, k, F0)
    assert np.allclose(b2.sumF, oracle.colsum(F0), rtol=1e-13)
    b.close(); b2.close()


def test_loglikelihood_and_fused_identity(oracle):
    n, k = 600, 20
    rp, col = random_graph(n, 7, seed=33, hub=100)
    rng = np.random.default_rng(33)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.3)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    b = _solver(rp, col, k, F0, sumF)
    assert abs(b.loglikelihood() - oracle.llh(rp, col, F0, sumF, P)) <= 1e-11 * abs(oracle.llh(rp, col, F0, sumF, P))
    llh1 = b.backtrackingLineSearchs()
    assert abs(b.loglikelihood() - llh1) <= 1e-12 * abs(llh1)     # LLH(t) == standalone LLH of the new state
    b.close()


@pytest.mark.parametrize("variant", [4, 3, 2])
def test_run_loop_matches_oracle(oracle, variant):
    n, k = 400, 8
    rp, col = random_graph(n, 6, seed=41)
    rng = np.random.default_rng(41)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.4)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    Fo, so, llho, callso, tro = oracle.run(rp, col, F0, sumF, P, variant=variant)
    b = _solver(rp, col, k, F0, sumF)
    if variant == 4:
        ret = b.SGDFindC()
    else:
        b.MBSGD(version=variant)
        ret = b.last_trace[-1]
    assert b.last_calls == callso
    assert np.allclose(b.last_trace, tro, rtol=1e-9)
    assert abs(ret - llho) <= 1e-9 * abs(llho)
    scale = np.abs(Fo).max()
    assert np.abs(b.F - Fo).max() <= RTOL_F * scale
    assert np.allclose(b.sumF, so, rtol=1e-8)
    # capped run: exactly max_outer calls, state after that many calls
    b.set_F(F0, sumF=sumF)
    b._run(variant, 1e-4, 3)
    Fm, sm, llhm, callsm, trm = oracle.run(rp, col, F0, sumF, P, variant=variant, max_outer=3)
    if callsm == 3:
        assert b.last_calls == 3 and np.allclose(b.last_trace, trm, rtol=1e-9)
        assert np.abs(b.F - Fm).max() <= RTOL_F * np.abs(Fm).max()
    b.close()


def test_email_enron_k50_one_step(oracle, graphs):
    rp, col, _ = graphs.load_npz_graph("email-enron")
    n, K = len(rp) - 1, 50
    assert n == 36692 and len(col) == 367662
    F0 = graphs.synthetic_F0(n, K, seed=1234, density=0.05)
    sumF = oracle.colsum(F0)
    b = _solver(rp, col, K, F0, sumF)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, sumF, oracle.make_params(K))
    _check_step(b, r, llh, max_flips=3, where="enron", inputs=(rp, col, F0, sumF, oracle.make_params(K)))
    b.close()


def test_com_amazon_k200_steps_and_properties(oracle, graphs):
    """BASELINE config 3 at full size: two steps against the oracle, then size-independent
    properties over a longer run (Jacobi invariants, sumF drift, monotone step bookkeeping)."""
    rp, col, _ = graphs.load_npz_graph("com-amazon")
    n, K = len(rp) - 1, 200
    assert n == 334863 and len(col) == 1851744 and np.diff(rp).max() == 549
    F0 = graphs.synthetic_F0(n, K, seed=1234, density=0.05)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(K)
    b = _solver(rp, col, K, F0, sumF)
    F, s = F0, sumF
    for it in range(2):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P)
        _check_step(b, r, llh, max_flips=5, where=f"amazon it{it}", inputs=(rp, col, F, s, P))
        F, s = b.F, b.sumF
    # property (iii): incremental sumF stays within 1e-9 of the true column sums
    b._run(4, 0.0, 10)
    Fg, sg = b.F, b.sumF
    assert np.abs(sg - Fg.sum(axis=0)).max() <= 1e-9 * np.abs(sg).max()
    # property (i): LLH trace entry t == standalone loglikelihood of the state after t calls
    assert abs(b.loglikelihood() - b.last_trace[-1]) <= 1e-12 * abs(b.last_trace[-1])
    b.close()


def test_reference_style_init_then_steps(oracle, graphs):
    """F0 from conductanceLocalMin + initNeighborComF (bigclam4-7.scala:58-108), then the hot path: the sparse
    0/1 start exercises the x == 0 shortcut (p clamped to MAX_P_) and rows that grow from zero."""
    from bigclam_apachespark_b200 import BigClam
    rp, col, _ = graphs.load_npz_graph("facebook_combined")
    K = 10
    b = BigClam(record_accepted=True)
    b.set_graph(rp, col)
    F = b.initNeighborComF(K)
    assert set(np.unique(F)) <= {0.0, 1.0} and np.array_equal(b.sumF, F.sum(axis=0))
    sumF = oracle.colsum(F)
    P = oracle.make_params(K)
    for it in range(4):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, sumF, P)
        _check_step(b, r, llh, max_flips=2, where=f"ref-init it{it}", max_idx_diff=0.05, inputs=(rp, col, F, sumF, P))
        F, sumF = b.F, b.sumF
    b.close()


def test_k_sweep_driver(oracle):
    """The K sweep of bigclam4-7.scala:244-266 on a small graph against an ORACLE-DRIVEN sweep: the same K grid, the
    same reference-style F0 per K (NumPy twin of initNeighborComF), SGDFindC by the CPU restatement, the same stop rule
    (`1 - LLH_K / LLH_prev < 0.001`, LLHKold starting at 0.0 as coded)."""
    from bigclam_apachespark_b200 import BigClam
    from oracle import numpy_twin as T
    rp, col = random_graph(400, 6, seed=3, hub=30)
    b = BigClam(minCom=4, maxCom=16, divCom=4)
    b.set_graph(rp, col)
    assert b.Kset() == [4, 5, 7, 9, 12, 16]
    KforC, hist = b.sweep_K(max_outer=30)
    assert len(hist) >= 2 and [k for k, _ in hist] == b.Kset()[:len(hist)]
    if KforC:
        assert KforC == hist[-1][0] and (1 - hist[-1][1] / hist[-2][1]) < 0.001
    # the oracle's sweep
    ranked, _ = T.conductance_local_min(rp, col)
    assert np.array_equal(b.Sbc, ranked)
    LLHKold, K_o, hist_o = 0.0, 0, []
    for K in b.Kset():
        F0 = T.init_neighbor_com_F(rp, col, K, ranked)                       # (K <= number of candidates: no random padding)
        _, _, llh, calls, _ = oracle.run(rp, col, F0, oracle.colsum(F0), oracle.make_params(K), variant=4, rel_tol=1e-4, max_outer=30)
        hist_o.append((K, llh))
        with np.errstate(divide="ignore", invalid="ignore"):
            gain = 1.0 - np.float64(llh) / np.float64(LLHKold)
        if gain < 0.001:
            K_o = K
            break
        LLHKold = llh
    assert KforC == K_o and len(hist) == len(hist_o)
    for (k1, l1), (k2, l2) in zip(hist, hist_o):
        assert k1 == k2 and abs(l1 - l2) <= 1e-8 * abs(l2), (k1, l1, l2)
    b.close()


def test_rmat_skewed_graph(oracle, graphs):
    """R-MAT (a,b,c,d) = (.57,.19,.19,.05): a degree-1390 hub (block-cooperative hub phase, > 32 active
    components) and ~20 % isolated nodes."""
    rp, col = graphs.rmat_graph(5000, 50000, seed=42)
    n, k = len(rp) - 1, 24
    assert np.diff(rp).max() > 1000 and (np.diff(rp) == 0).sum() > 500
    F0 = graphs.synthetic_F0(n, k, seed=3, density=0.15)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    b = _solver(rp, col, k, F0, sumF)
    F, s = F0, sumF
    for it in range(3):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P)
        _check_step(b, r, llh, max_flips=2, where=f"rmat it{it}", max_idx_diff=0.05, inputs=(rp, col, F, s, P))
        F, s = b.F, b.sumF
    b.close()


def test_mega_hub_split_over_blocks(oracle, graphs):
    """A hub above kHubSlice (384) edges is split into slices processed by different blocks (phases 1-3 of
    the hub phase, partial sums through global scratch); a star-like graph makes it dominate."""
    rp, col = random_graph(3000, 4, seed=8, hub=2500)           # node 0 has ~2500 neighbours
    assert np.diff(rp).max() > 2000
    n, k = len(rp) - 1, 16
    rng = np.random.default_rng(8)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.3)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    b = _solver(rp, col, k, F0, sumF)
    F, s = F0, sumF
    for it in range(4):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P)
        _check_step(b, r, llh, max_flips=2, where=f"mega it{it}", max_idx_diff=0.05, inputs=(rp, col, F, s, P))
        F, s = b.F, b.sumF
    # the device-side loop uses the same kernels
    b.set_F(F0, sumF=sumF)
    b._run(4, 1e-4, 12)
    Fo, so, llho, callso, tro = oracle.run(rp, col, F0, sumF, P, variant=4, max_outer=12)
    assert b.last_calls == callso and np.allclose(b.last_trace, tro, rtol=1e-8)
    b.close()


def test_step_speculation_is_invisible(oracle):
    """bigclam_step launches the next call's kernel speculatively (its PRE is this call's LLH).  Interleaving
    other entry points, changing the uset or resetting F must give exactly the non-speculative results."""
    n, k = 500, 10
    rp, col = random_graph(n, 6, seed=71, hub=80)
    rng = np.random.default_rng(71)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.4)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    b = _solver(rp, col, k, F0, sumF)
    F, s = F0, sumF
    masks = [None, None, rng.random(n) < 0.5, rng.random(n) < 0.5, None, None]
    for it, mk in enumerate(masks):
        uset = None if mk is None else np.flatnonzero(mk)
        llh = b.backtrackingLineSearchs(uset=uset)
        r = oracle.step(rp, col, F, s, P, node_mask=None if mk is None else mk.astype(np.uint8))
        _check_step(b, r, llh, max_flips=1, where=f"spec it{it}", max_idx_diff=0.05, inputs=(rp, col, F, s, P))
        if it == 1:
            assert abs(b.loglikelihood() - llh) <= 1e-12 * abs(llh)      # drops the speculation, state unchanged
        F, s = b.F, b.sumF
    # a reset in the middle of a speculated sequence
    b.set_F(F0, sumF=sumF)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, sumF, P)
    _check_step(b, r, llh, max_flips=1, where="spec after set_F", inputs=(rp, col, F0, sumF, P))
    # the device loop after speculative single steps
    b._run(4, 1e-4, 5)
    Fo, so, llho, callso, tro = oracle.run(rp, col, r.F, r.sumF, P, variant=4, max_outer=5)
    assert np.allclose(b.last_trace, tro, rtol=1e-8)
    b.close()
