"""Community scores (BigClam.community_stats) on one GPU, against the host route (F_csr() + the NumPy twin,
tests/community_stats_twin.py):

  amazon     com-amazon fitted at K = 200 (initNeighborComF + SGDFindC), delta of the script (count = vertices with
             edges), zero rows in every community and in none: both routes; the median conductance of the non-empty
             communities beside the Avg-F1 against com-amazon.cmty (printed, not asserted);
  K2000      com-amazon, synthetic F0 at K = 2000 after 2 steps: the GPU only (the host route would hold 33 M
             memberships in NumPy);
  K9000      the same at K = 9000 (145 M memberships): the GPU only;
  planted    a planted model with n = 10^6 and K = 1000 (every node in one community, 30 % in a second, F = 0.15) on the
             graph sampled from it (sample_graph, eps = 0): both routes.

GPU times are host clocks around synchronous calls, host buffers included, the best of --reps calls after a warm-up;
the host route is timed over one call.  Where both routes run, their arrays are compared bit for bit.  The card's name and power limit are read in the same run.

    python scripts/bench_community_stats.py [--out DIR] [--reps N]

Prints one JSON line (and writes it to DIR/bench_community_stats.json when --out is given)."""
import argparse
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "scripts"))
sys.dont_write_bytecode = True

from bench_extract import _best, _card  # noqa: E402


def _routes(b, delta, res, tag, reps, everywhere=True, host=True):
    from community_stats_twin import community_stats
    g, t = _best(lambda: b.community_stats(delta, everywhere), reps)
    res[f"{tag}_gpu_s"] = t
    res[f"{tag}_nonempty_communities"] = int((g["size"] > 0).sum())
    if not host:
        res[f"{tag}_host_route_s"] = "not run: the twin holds every membership on the host"
        return g
    t0 = time.perf_counter()                                # one call: minutes of host work would buy no precision
    h = community_stats(*b.F_csr(), b.K, delta, b.rowptr, b.col, zero_rows=everywhere)
    res[f"{tag}_host_route_s"] = time.perf_counter() - t0
    res[f"{tag}_routes_equal"] = bool(all(np.array_equal(np.asarray(g[k]).view(np.int64), np.asarray(h[k]).view(np.int64))
                                          for k in ("size", "volume", "internal", "conductance")))
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
    coded = Cm.delta_threshold(n, int((np.diff(rp) > 0).sum()))

    # com-amazon fitted at K = 200
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col)
    b.initNeighborComF(200)
    b.SGDFindC()
    truth = Cm.load_ground_truth()
    g = b.extract_communities(coded)
    res["amazon_zero_rows"] = int(len(g[2]))
    for everywhere in (True, False):
        tag = f"amazon_zero_rows_{'everywhere' if everywhere else 'nowhere'}"
        s = _routes(b, coded, res, tag, args.reps, everywhere)
        res[f"{tag}_median_conductance"] = float(np.median(s["conductance"][s["size"] > 0]))
        comms, _ = Cm.group(*g, zero_rows_everywhere=everywhere)
        res[f"{tag}_avg_f1"] = Cm.avg_f1(comms, truth, n)
    b.close()

    # com-amazon, synthetic F0 after 2 steps, K = 2000 and 9000
    for K in (2000, 9000):
        b = BigClam(sparse_rows=True)
        b.set_graph(rp, col).set_K(K).set_F_csr(*G.synthetic_F0_csr(n, K, seed=1234, density=0.05))
        for _ in range(2):
            b.backtrackingLineSearchs()
        _routes(b, coded, res, f"K{K}", args.reps, host=False)
        b.close()

    # planted, n = 10^6, K = 1000, on the graph sampled from it
    from bench_sample import _planted
    n, K = 1_000_000, 1000
    ip, ix, vl = _planted(n, K, 0.15, 0.3, seed=3)
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(ip, ix, vl)
    grp, gcol = b.sample_graph(seed=5)
    b.close()
    res["planted_entries"] = int(len(gcol))
    b = BigClam(sparse_rows=True)
    b.set_graph(grp, gcol).set_K(K).set_F_csr(ip, ix, vl)
    _routes(b, 0.1, res, "planted", args.reps)
    b.close()

    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_community_stats.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
