"""Edge probabilities and link recommendations on com-amazon: bigclam_pair_affinity over all directed edges (K = 200 and
2000), bigclam_recommend(m = 10) for all nodes (K = 200), and the host route (F_csr() plus the NumPy twin of
tests/links_twin.py) on the same work.  F is the bench's synthetic F0 (density 0.05) after a few steps.  Times are host
clocks around calls that end in a stream synchronise; the card's name and power limit are read in the same run.

    python scripts/bench_links.py [--out DIR] [--host-nodes N]

Prints one JSON line (and writes it to DIR/bench_links.json when --out is given)."""
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
    fn()                                                    # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-nodes", type=int, default=20000, help="query nodes of the host route's recommendation")
    args = ap.parse_args()
    from bigclam_apachespark_b200 import BigClam, graphs as G
    from links_twin import Twin

    rp, col, _ = G.load_npz_graph("com-amazon")
    n = len(rp) - 1
    u = np.repeat(np.arange(n, dtype=np.int32), np.diff(rp))
    res = {"card": _card(), "graph": "com-amazon", "n": n, "directed_edges": int(len(col))}
    for K, steps in ((200, 3), (2000, 2)):
        b = BigClam(sparse_rows=True)
        b.set_graph(rp, col).set_K(K).set_F_csr(*G.synthetic_F0_csr(n, K, seed=1234, density=0.05))
        for _ in range(steps):
            b.backtrackingLineSearchs()
        t, ts = _best(lambda: b.edge_probability(u, col), args.reps)
        res[f"pairs_K{K}_s"] = t
        res[f"pairs_K{K}_per_s"] = len(col) / t
        # host route: download the rows, then the twin
        t0 = time.perf_counter()
        tw = Twin(*b.F_csr(), K)
        step = 1 << 18                                      # (bounded host memory at K = 2000)
        xh = np.concatenate([tw.x(u[i:i + step], col[i:i + step]) for i in range(0, len(col), step)])
        res[f"host_pairs_K{K}_s"] = time.perf_counter() - t0
        xd, _ = b.edge_probability(u, col)
        res[f"pairs_K{K}_bit_identical"] = bool(np.array_equal(xd.view(np.int64), xh.view(np.int64)))
        if K == 200:
            t, ts = _best(lambda: b.recommend(None, 10), max(1, args.reps // 2))
            res["recommend_K200_m10_all_s"] = t
            res["recommend_K200_m10_nodes_per_s"] = n / t
            q = np.arange(min(n, args.host_nodes))
            t0 = time.perf_counter()
            tw = Twin(*b.F_csr(), K)
            hv, hx, _ = tw.recommend(rp, col, q, 10)
            th = time.perf_counter() - t0
            res["host_recommend_nodes"] = len(q)
            res["host_recommend_s"] = th
            res["host_recommend_nodes_per_s"] = len(q) / th
            dv, dx = b.recommend(q, 10)
            res["recommend_matches_host"] = bool(np.array_equal(dv, hv) and np.array_equal(dx.view(np.int64), hx.view(np.int64)))
        b.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_links.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
