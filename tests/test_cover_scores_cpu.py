"""The NumPy twin of the cover scores (tests/cover_scores_twin.py) on its own: hand-computed covers in both zero-row
modes (an empty truth community, repeated and unsorted truth ids, a community of all n nodes), Avg-F1 against
communities.avg_f1, both NMIs against a pure-Python evaluation over node sets, and the self-score of exactly 1.0."""
import numpy as np
import pytest
import scipy.sparse as sp

from cover_scores_twin import KEYS, cover_scores, nmi_by_sets
from extract_twin import extract_grouped


def _csr(rows):
    indptr = np.cumsum([0] + [len(r) for r in rows]).astype(np.int64)
    indices = np.array([c for r in rows for c in sorted(r)], dtype=np.int32)
    values = np.array([r[c] for r in rows for c in sorted(r)], dtype=np.float64)
    return indptr, indices, values


def _f1(a, s):
    return (2.0 * a) / s


# X_0 = {0, 1, 5} (row 5 by its maximum below delta), X_1 = {1, 2, 3}, X_2 = {}; row 4 is all zero.
HAND_F = _csr([{0: 1.0}, {0: 1.0, 1: 1.0}, {1: 1.0}, {1: 1.0}, {}, {0: 0.2}])
# Y_0 = {1, 2, 3} given unsorted with a repeat, Y_1 empty, Y_2 all six nodes, Y_3 = {0, 5}
HAND_TRUTH = [np.array([3, 2, 2, 1]), np.array([], dtype=np.int64), np.arange(6)[::-1], np.array([5, 0])]


def test_hand_cover_zero_rows_nowhere():
    g = cover_scores(*HAND_F, 3, 0.5, HAND_TRUTH, zero_rows=False)
    # X_0: Y_0 a=1 -> 2/6, Y_2 a=3 -> 6/9, Y_3 a=2 -> 4/5.  X_1: Y_0 a=3 -> 1, Y_2 -> 6/9, Y_3 a=0.  X_2 empty.
    assert g["f1_detected"].tolist() == [_f1(2, 5), _f1(3, 6), 0.0]
    assert g["match_detected"].tolist() == [3, 0, -1]
    # Y_2 ties between X_0 and X_1 at 6/9: the smaller id
    assert g["f1_truth"].tolist() == [_f1(3, 6), 0.0, _f1(3, 9), _f1(2, 5)]
    assert g["match_truth"].tolist() == [1, -1, 0, 0]
    assert g["avg_f1"] == 0.5 * ((_f1(2, 5) + _f1(3, 6)) / 2 + (((_f1(3, 6) + 0.0) + _f1(3, 9)) + _f1(2, 5)) / 4)
    # X_1 = Y_0: the self pair is exactly 0; the empty X_2, the empty Y_1 and the full Y_2 are outside the NMI
    assert g["hcond_detected"][1] == 0.0 and g["hcond_truth"][0] == 0.0
    assert np.isnan(g["hcond_detected"][2]) and np.isnan(g["hcond_truth"][1]) and np.isnan(g["hcond_truth"][2])
    lfk, mx = nmi_by_sets([[0, 1, 5], [1, 2, 3]], HAND_TRUTH, 6)
    assert g["nmi_lfk"] == pytest.approx(lfk, rel=1e-12, abs=1e-15)
    assert g["nmi_max"] == pytest.approx(mx, rel=1e-12, abs=1e-15)


def test_hand_cover_zero_rows_everywhere():
    g = cover_scores(*HAND_F, 3, 0.5, HAND_TRUTH, zero_rows=True)
    # X_0 = {0, 1, 4, 5}: Y_0 a=1 -> 2/7, Y_2 a=4 -> 8/10, Y_3 a=2 -> 4/6.  X_1 = {1, 2, 3, 4}: Y_0 a=3 -> 6/7, Y_2 8/10.
    # X_2 = {4}: Y_2 a=1 -> 2/7.
    assert g["f1_detected"].tolist() == [_f1(4, 10), _f1(3, 7), _f1(1, 7)]
    assert g["match_detected"].tolist() == [2, 0, 2]
    assert g["f1_truth"].tolist() == [_f1(3, 7), 0.0, _f1(4, 10), _f1(2, 6)]
    assert g["match_truth"].tolist() == [1, -1, 0, 0]
    lfk, mx = nmi_by_sets([[0, 1, 4, 5], [1, 2, 3, 4], [4]], HAND_TRUTH, 6)
    assert g["nmi_lfk"] == pytest.approx(lfk, rel=1e-12, abs=1e-15)
    assert g["nmi_max"] == pytest.approx(mx, rel=1e-12, abs=1e-15)


def test_hand_nmi_value():
    """X = {{0, 1}}, Y = {{0, 1}, {2, 3}} on n = 4, written out: the pair (X_0, Y_0) is the self pair (0); (X_0, Y_1) has
    a = 0 and h(0) + h(0) > h(2) + h(2) fails, so H*(Y_1 | X) = H(Y_1) = 2 h(2) with h(2) = -(0.5 ln 0.5)."""
    F = _csr([{0: 1.0}, {0: 1.0}, {}, {}])
    g = cover_scores(*F, 1, 0.5, [[0, 1], [2, 3]], zero_rows=False)
    h2 = -(0.5 * np.log(0.5))
    assert g["hcond_detected"].tolist() == [0.0]
    assert g["hcond_truth"].tolist() == [0.0, h2 + h2]
    assert g["nmi_lfk"] == 1.0 - 0.5 * (0.0 + (0.0 + 1.0) / 2)
    assert g["nmi_max"] == 0.5 * ((2 * h2 - 0.0) + ((2 * h2 + 2 * h2) - (0.0 + 2 * h2))) / (4 * h2)


def _random_case(seed, n=80, K=9):
    rng = np.random.default_rng(seed)
    F = rng.random((n, K)) * (rng.random((n, K)) < 0.3)
    F[::7] = 0.0
    F[3, :3] = 0.25
    m = sp.csr_matrix(F)
    truth = [rng.choice(n, size=int(rng.integers(1, n // 3)), replace=False) for _ in range(12)]
    return (m.indptr, m.indices, m.data), K, truth, rng


def _detected(F, K, delta, everywhere):
    from bigclam_apachespark_b200 import communities as Cm
    return Cm.group(*extract_grouped(*F, K, delta), zero_rows_everywhere=everywhere)


@pytest.mark.parametrize("everywhere", [True, False])
@pytest.mark.parametrize("delta", [0.1, 0.5, float("inf")])
def test_avg_f1_matches_communities_avg_f1(everywhere, delta):
    from bigclam_apachespark_b200 import communities as Cm
    for seed in range(4):
        F, K, truth, _ = _random_case(seed)
        n = len(F[0]) - 1
        truth = truth + [np.zeros(0, dtype=np.int64)]                             # an empty truth community counts with 0
        g = cover_scores(*F, K, delta, truth, zero_rows=everywhere)
        det, _ = _detected(F, K, delta, everywhere)
        assert g["avg_f1"] == pytest.approx(Cm.avg_f1(det, truth, n), rel=1e-12, abs=0), (seed, delta)


@pytest.mark.parametrize("everywhere", [True, False])
@pytest.mark.parametrize("delta", [0.1, 0.5, float("inf")])
def test_nmi_matches_sets(everywhere, delta):
    for seed in range(4):
        F, K, truth, rng = _random_case(seed)
        n = len(F[0]) - 1
        truth = truth + [np.arange(n), np.zeros(0, dtype=np.int64), rng.integers(0, n, 30)]   # all n, empty, repeats
        g = cover_scores(*F, K, delta, truth, zero_rows=everywhere)
        det, _ = _detected(F, K, delta, everywhere)
        lfk, mx = nmi_by_sets(det, truth, n)
        assert g["nmi_lfk"] == pytest.approx(lfk, rel=1e-12, abs=1e-15), (seed, delta)
        assert g["nmi_max"] == pytest.approx(mx, rel=1e-12, abs=1e-15), (seed, delta)


@pytest.mark.parametrize("everywhere", [True, False])
def test_self_score_is_one(everywhere):
    for seed in range(4):
        F, K, _, _ = _random_case(seed)
        for delta in (0.1, 0.5, float("inf")):
            det, cids = _detected(F, K, delta, everywhere)
            g = cover_scores(*F, K, delta, det, zero_rows=everywhere)
            assert (g["avg_f1"], g["nmi_lfk"], g["nmi_max"]) == (1.0, 1.0, 1.0), (seed, delta)
            first = {}                                                      # coinciding communities match the first
            for i, c in enumerate(det):
                first.setdefault(c.tobytes(), i)
            want = np.array([first[c.tobytes()] for c in det])
            assert np.array_equal(g["match_detected"][cids], want)
            assert np.array_equal(g["match_truth"], cids[want])


def test_truth_order_and_repeats_do_not_matter():
    F, K, truth, rng = _random_case(11)
    a = cover_scores(*F, K, 0.5, truth)
    shuffled = [np.concatenate([rng.permutation(t), t[: len(t) // 2]]) for t in truth]
    b = cover_scores(*F, K, 0.5, shuffled)
    for key in KEYS:
        assert np.array_equal(np.asarray(a[key]).view(np.uint8), np.asarray(b[key]).view(np.uint8)), key
    assert (a["avg_f1"], a["nmi_lfk"], a["nmi_max"]) == (b["avg_f1"], b["nmi_lfk"], b["nmi_max"])
