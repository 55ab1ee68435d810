"""Cover scores (BigClam.score_against: Avg-F1 and overlapping NMI against a known cover) on one GPU, against the host
route (extract_communities + communities.group + communities.avg_f1, and the NumPy twin tests/cover_scores_twin.py for
the NMI):

  amazon     com-amazon fitted at K = 200 (initNeighborComF + SGDFindC), delta of the script (count = vertices with
             edges), against com-amazon.cmty, zero rows in every community and in none: both routes, their F1 arrays and
             matches compared bit for bit and the scores side by side;
  K2000      com-amazon, synthetic F0 at K = 2000 after 2 steps, against com-amazon.cmty: the GPU only;
  K9000      the same at K = 9000: the GPU only;
  planted    a planted model with n = 10^6 and K = 1000 (every node in one community, 30 % in a second, F = 0.15)
             against its planted communities: the GPU only; every score should be exactly 1.

GPU times are host clocks around synchronous calls, host buffers included (the truth lists are packed into a CSR on
every call), the best of --reps calls after a warm-up; the host route is timed over one call.  The card's name and power
limit are read in the same run.

    python scripts/bench_cover_scores.py [--out DIR] [--reps N]

Prints one JSON line (and writes it to DIR/bench_cover_scores.json when --out is given)."""
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

SCALARS = ("avg_f1", "nmi_lfk", "nmi_max")


def _gpu(b, truth, delta, res, tag, reps, everywhere=True):
    g, t = _best(lambda: b.score_against(truth, delta, everywhere), reps)
    res[f"{tag}_gpu_s"] = t
    for k in SCALARS:
        res[f"{tag}_{k}"] = g[k]
    res[f"{tag}_pairs"] = int(b.K) * len(truth)
    return g


def _host(b, truth, delta, g, res, tag, everywhere):
    from bigclam_apachespark_b200 import communities as Cm
    from cover_scores_twin import cover_scores
    t0 = time.perf_counter()                                # one call: seconds of host work would buy no precision
    det, _ = Cm.group(*b.extract_communities(delta), zero_rows_everywhere=everywhere)
    avg = Cm.avg_f1(det, truth, b.n)
    h = cover_scores(*b.F_csr(), b.K, delta, truth, zero_rows=everywhere)
    res[f"{tag}_host_route_s"] = time.perf_counter() - t0
    res[f"{tag}_host_avg_f1"] = avg
    res[f"{tag}_host_nmi_lfk"] = h["nmi_lfk"]
    res[f"{tag}_host_nmi_max"] = h["nmi_max"]
    res[f"{tag}_f1_and_matches_equal"] = bool(all(np.array_equal(np.asarray(g[k]).view(np.uint8), np.asarray(h[k]).view(np.uint8))
                                                  for k in ("f1_detected", "match_detected", "f1_truth", "match_truth")))
    res[f"{tag}_max_hcond_diff"] = float(max(np.nanmax(np.abs(g[k] - h[k])) for k in ("hcond_detected", "hcond_truth")))
    res[f"{tag}_admissibility_margin"] = h["margin"]


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
    truth = Cm.load_ground_truth()
    res["amazon_truth_communities"] = len(truth)

    # com-amazon fitted at K = 200
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col)
    b.initNeighborComF(200)
    b.SGDFindC()
    for everywhere in (True, False):
        tag = f"amazon_zero_rows_{'everywhere' if everywhere else 'nowhere'}"
        g = _gpu(b, truth, coded, res, tag, args.reps, everywhere)
        _host(b, truth, coded, g, res, tag, everywhere)
    b.close()

    # com-amazon, synthetic F0 after 2 steps, K = 2000 and 9000
    for K in (2000, 9000):
        b = BigClam(sparse_rows=True)
        b.set_graph(rp, col).set_K(K).set_F_csr(*G.synthetic_F0_csr(n, K, seed=1234, density=0.05))
        for _ in range(2):
            b.backtrackingLineSearchs()
        _gpu(b, truth, coded, res, f"K{K}", args.reps)
        b.close()

    # planted, n = 10^6, K = 1000, against its planted communities
    from bench_sample import _planted
    n, K = 1_000_000, 1000
    ip, ix, vl = _planted(n, K, 0.15, 0.3, seed=3)
    rows = np.repeat(np.arange(n, dtype=np.int32), np.diff(ip))
    o = np.argsort(ix, kind="stable")
    planted = np.split(rows[o], np.cumsum(np.bincount(ix, minlength=K))[:-1])
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(ip, ix, vl)
    g = _gpu(b, planted, 0.1, res, "planted", args.reps)
    res["planted_all_one"] = all(g[k] == 1.0 for k in SCALARS)
    b.close()

    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_cover_scores.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
