"""Graphs sampled from the model (BigClam.sample_graph) on one GPU:

  amazon    com-amazon fitted at K = 200 (initNeighborComF + SGDFindC), sampled with eps = 0 and eps = 1 - MAX_P_: wall
            time of a sample with host buffers (count + fill calls), the co-member pairs the rows examine
            (sum_c |M_c| (|M_c| - 1), M_c = the nodes with F_uc != 0), sampled edges against the input's; the NumPy twin
            (tests/sample_twin.py) on a few rows, checked against the device's rows and extrapolated to all rows;
  planted   a planted model with n = 10^6 and K = 1000 on isolated nodes (set_F_csr), same measurements;
  recover   a planted model (n = 20000, K = 100) -> sample -> initNeighborComF + SGDFindC -> extract -> Avg-F1 against
            the planted communities (printed, not asserted).

Times are host clocks around calls that end in a stream synchronise; the card's name and power limit are read in the
same run.

    python scripts/bench_sample.py [--out DIR] [--reps N] [--twin-rows N]

Prints one JSON line (and writes it to DIR/bench_sample.json when --out is given)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.dont_write_bytecode = True


def _card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                  # noqa: BLE001
        return f"unknown ({e})"


def _best(fn, reps):
    out = fn()                                              # warm-up (and the result)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return out, min(ts)


def _planted(n, K, fval, extra, seed):
    """Node u in community u * K // n (F = fval), and with probability `extra` in one more random community."""
    rng = np.random.default_rng(seed)
    c0 = (np.arange(n, dtype=np.int64) * K) // n
    two = rng.random(n) < extra
    c1 = rng.integers(0, K, n)
    two &= c1 != c0
    cnt = 1 + two.astype(np.int64)
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(cnt, out=indptr[1:])
    lo, hi = np.minimum(c0, c1), np.maximum(c0, c1)
    first = np.where(two, lo, c0)
    indices = np.empty(indptr[-1], dtype=np.int32)
    indices[indptr[:-1]] = first
    indices[indptr[:-1][two] + 1] = hi[two]
    values = np.full(indptr[-1], float(fval))
    return indptr, indices, values


def _measure(b, res, tag, real_edges, reps, twin_rows):
    from sample_twin import SampleTwin
    ip, ix, vl = b.F_csr()
    m = np.bincount(ix, minlength=b.K).astype(np.float64)
    res[f"{tag}_comember_pairs"] = float((m * (m - 1)).sum())
    for name, eps in (("eps0", 0.0), ("epsfloor", 1.0 - b.MAX_P_)):
        (rp, col), t = _best(lambda: b.sample_graph(seed=1, eps=eps), reps)
        res[f"{tag}_{name}_s"] = t
        res[f"{tag}_{name}_edges"] = int(len(col) // 2)
        if real_edges is not None:
            res[f"{tag}_{name}_edges_over_real"] = len(col) / 2 / real_edges
        if twin_rows and name == "epsfloor":
            tw = SampleTwin(ip, ix, vl, b.K, b.MIN_P_, b.MAX_P_)
            rows = np.linspace(0, b.n - 1, twin_rows).astype(np.int64)
            t0 = time.perf_counter()
            ok = all(np.array_equal(tw.row(int(u), 1, eps), col[rp[u]:rp[u + 1]]) for u in rows)
            tt = time.perf_counter() - t0
            res[f"{tag}_twin_rows"] = int(twin_rows)
            res[f"{tag}_twin_s_per_row"] = tt / twin_rows
            res[f"{tag}_twin_all_rows_s_extrapolated"] = tt / twin_rows * b.n
            res[f"{tag}_twin_rows_match"] = bool(ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--twin-rows", type=int, default=8)
    args = ap.parse_args()
    from bigclam_apachespark_b200 import BigClam, communities as Cm, graphs as G

    res = {"card": _card()}
    # com-amazon, fitted at K = 200
    rp, col, _ = G.load_npz_graph("com-amazon")
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col)
    t0 = time.perf_counter()
    b.initNeighborComF(200)
    b.SGDFindC()
    res["amazon_fit_s"] = time.perf_counter() - t0
    res["amazon_n"], res["amazon_edges"] = b.n, int(len(col) // 2)
    _measure(b, res, "amazon", len(col) // 2, args.reps, args.twin_rows)
    b.close()

    # planted, n = 10^6, K = 1000 (communities of 1000, 30 % of the nodes in a second one, F = 0.15: p_in = 0.022)
    n, K = 1_000_000, 1000
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K)
    b.set_F_csr(*_planted(n, K, 0.15, 0.3, seed=3))
    res["planted_n"], res["planted_K"] = n, K
    _measure(b, res, "planted", None, args.reps, max(1, args.twin_rows // 4))
    b.close()

    # planted -> sample -> fit -> extract -> Avg-F1 against the planted communities
    n, K = 20000, 100
    ip, ix, vl = _planted(n, K, 0.6, 0.3, seed=4)
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(ip, ix, vl)
    srp, scol = b.sample_graph(seed=5, eps=1.0 - b.MAX_P_)
    b.close()
    owner = np.repeat(np.arange(n, dtype=np.int32), np.diff(ip))
    truth = [owner[ix == c] for c in range(K)]
    f = BigClam(sparse_rows=True)
    f.set_graph(srp, scol)
    t0 = time.perf_counter()
    f.initNeighborComF(K)
    f.SGDFindC()
    res["recover_n"], res["recover_K"], res["recover_edges"] = n, K, int(len(scol) // 2)
    res["recover_fit_s"] = time.perf_counter() - t0
    for rule, cnt in (("coded", int((np.diff(srp) > 0).sum())), ("thesis", len(scol) // 2)):
        comms, _, _ = Cm.extract(f, Cm.delta_threshold(n, cnt))
        res[f"recover_avg_f1_{rule}"] = Cm.avg_f1(comms, truth, n)
        res[f"recover_communities_{rule}"] = len(comms)
    f.close()

    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sample.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
