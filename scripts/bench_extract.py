"""Communities grouped by community (BigClam.extract_communities) on one GPU, against the dense route
(communities.extract: bigclam_extract's n x K member bytes, regrouped on the host) and the host route (F_csr() + the
NumPy twin, tests/extract_twin.py):

  amazon     com-amazon fitted at K = 200 (initNeighborComF + SGDFindC), delta of the script (count = vertices with
             edges): the three routes; zero rows, non-empty communities, memberships; Avg-F1 against com-amazon.cmty for
             both deltas (coded and thesis), with the zero rows in every community or in none (printed, not asserted);
  K2000      com-amazon, synthetic F0 at K = 2000 after 2 steps: grouped and dense route;
  K9000      the same at K = 9000: grouped (the dense route only when its n x K host bytes stay under 2 GiB);
  planted    a planted model with n = 10^6 and K = 1000 on isolated nodes (set_F_csr): grouped, and whether the
             communities are exactly the planted ones.

Times are host clocks around synchronous calls, host buffers included, the best of --reps calls after a warm-up.  The
arrays of every route that runs are compared.  The card's name and power limit are read in the same run.

    python scripts/bench_extract.py [--out DIR] [--reps N]

Prints one JSON line (and writes it to DIR/bench_extract.json when --out is given)."""
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


def _same_lists(a, b):
    return len(a[0]) == len(b[0]) and np.array_equal(a[1], b[1]) and all(np.array_equal(x, y) for x, y in zip(a[0], b[0]))


def _routes(b, delta, res, tag, reps, dense=True, host=False):
    from bigclam_apachespark_b200 import communities as Cm
    from extract_twin import extract_grouped
    g, t = _best(lambda: b.extract_communities(delta), reps)
    res[f"{tag}_grouped_s"] = t
    res[f"{tag}_memberships"] = int(len(g[1]))
    res[f"{tag}_zero_rows"] = int(len(g[2]))
    res[f"{tag}_nonempty_communities"] = int((np.diff(g[0]) > 0).sum())
    same = True
    if dense:
        d, t = _best(lambda: Cm.extract(b, delta), reps)
        res[f"{tag}_dense_route_s"] = t
        same &= _same_lists((d[0], d[1]), Cm.group(*g))
    else:
        res[f"{tag}_dense_route_s"] = f"skipped: {b.n} x {b.K} host bytes"
    if host:
        h, t = _best(lambda: extract_grouped(*b.F_csr(), b.K, delta), reps)
        res[f"{tag}_host_route_s"] = t
        same &= all(np.array_equal(x, y) for x, y in zip(g, h))
    res[f"{tag}_routes_equal"] = bool(same)
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from bigclam_apachespark_b200 import BigClam, communities as Cm, graphs as G

    res = {"card": _card()}
    rp, col, _ = G.load_npz_graph("com-amazon")
    n = len(rp) - 1
    res["amazon_n"] = n
    coded = Cm.delta_threshold(n, int((np.diff(rp) > 0).sum()))
    thesis = Cm.delta_threshold(n, len(col) // 2)

    # com-amazon fitted at K = 200
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col)
    t0 = time.perf_counter()
    b.initNeighborComF(200)
    b.SGDFindC()
    res["amazon_fit_s"] = time.perf_counter() - t0
    _routes(b, coded, res, "amazon", args.reps, dense=True, host=True)
    truth = Cm.load_ground_truth()
    for rule, delta in (("coded", coded), ("thesis", thesis)):
        g = b.extract_communities(delta)
        for everywhere in (True, False):
            comms, _ = Cm.group(*g, zero_rows_everywhere=everywhere)
            res[f"amazon_avg_f1_{rule}_zero_rows_{'everywhere' if everywhere else 'nowhere'}"] = Cm.avg_f1(comms, truth, n)
    b.close()

    # com-amazon, synthetic F0 after 2 steps, K = 2000 and 9000
    for K in (2000, 9000):
        b = BigClam(sparse_rows=True)
        b.set_graph(rp, col).set_K(K).set_F_csr(*G.synthetic_F0_csr(n, K, seed=1234, density=0.05))
        for _ in range(2):
            b.backtrackingLineSearchs()
        _routes(b, coded, res, f"K{K}", args.reps, dense=n * K < (1 << 31))
        b.close()

    # planted, n = 10^6, K = 1000
    from bench_sample import _planted
    n, K = 1_000_000, 1000
    ip, ix, vl = _planted(n, K, 0.15, 0.3, seed=3)
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(ip, ix, vl)
    g = _routes(b, 0.1, res, "planted", args.reps, dense=False)
    owner = np.repeat(np.arange(n, dtype=np.int32), np.diff(ip))
    o = np.lexsort((owner, ix))
    res["planted_exact"] = bool(len(g[2]) == 0 and np.array_equal(g[1], owner[o])
                                and np.array_equal(g[0][1:], np.cumsum(np.bincount(ix, minlength=K))))
    b.close()

    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_extract.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
