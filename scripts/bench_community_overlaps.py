"""Community overlaps (BigClam.community_overlaps: the shared members of every overlapping pair of communities) on one
GPU, against the host route (F_csr() + the NumPy twin tests/community_overlaps_twin.py, M^T M in SciPy):

  amazon     com-amazon fitted at K = 200 (initNeighborComF + SGDFindC), delta of the script (count = vertices with
             edges), zero rows in every community and in none: both routes, their arrays compared bit for bit;
  K2000      com-amazon, synthetic F0 at K = 2000 after 2 steps: the GPU only;
  K9000      the same at K = 9000: the GPU only;
  planted    a planted model with n = 10^6 and K = 1000 (every node in one community, 30 % in a second, F = 0.15), as
             in bench_sample.py: both routes.

For each workload: the work of one pass, sum over the non-zero rows u of m_u^2 (m_u = the communities u is in), and
the largest per-community share of it (sum over u in M_c of m_u, the work of one block); nnz; and the number of pairs
{c, d} with Jaccard >= 0.5 in both zero-row modes (as coded, a pair that is not listed still shares the z zero rows
and is counted when z / (size_c + size_d - z) >= 0.5).  GPU times are host clocks around synchronous calls, host
buffers included (the count call and the fill call), the best of --reps calls after a warm-up; the host route is timed
over one call.  The card's name and power limit are read in the same run.

    python scripts/bench_community_overlaps.py [--out DIR] [--reps N]

Prints one JSON line (and writes it to DIR/bench_community_overlaps.json when --out is given)."""
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


def _jaccard_pairs(g, everywhere):
    """Pairs {c, d} with Jaccard >= 0.5, the unlisted pairs of the as-coded mode included."""
    listed = int((g["jaccard"] >= 0.5).sum()) // 2
    z = g["zero_rows"] if everywhere else 0
    if z == 0:
        return listed
    s = np.sort(g["size"])                                   # an unlisted pair: z / (s_c + s_d - z) >= 0.5 iff s_c + s_d <= 3 z
    K = len(s)
    within = int((np.searchsorted(s, 3 * z - s, side="right") - (2 * s <= 3 * z)).sum()) // 2
    rows = np.repeat(np.arange(K), np.diff(g["ptr"]))
    size = g["size"]
    listed_within = int((size[rows] + size[g["other"]] <= 3 * z).sum()) // 2
    return within - listed_within + listed


def _work(b, delta, res, tag):
    comptr, members, _ = b.extract_communities(delta)
    m = np.bincount(members, minlength=b.n).astype(np.int64)
    res[f"{tag}_pass_increments"] = int((m * m).sum())
    per_c = np.add.reduceat(np.append(m[members], 0), comptr[:-1]) * (np.diff(comptr) > 0)
    res[f"{tag}_largest_block_increments"] = int(per_c.max()) if len(per_c) else 0


def _gpu(b, delta, res, tag, reps, everywhere=True):
    g, t = _best(lambda: b.community_overlaps(delta, 1, everywhere), reps)
    res[f"{tag}_gpu_s"] = t
    res[f"{tag}_nnz"] = int(g["ptr"][-1])
    res[f"{tag}_zero_rows"] = g["zero_rows"]
    res[f"{tag}_jaccard_ge_half_pairs"] = _jaccard_pairs(g, everywhere)
    return g


def _host(b, delta, g, res, tag, everywhere):
    from community_overlaps_twin import community_overlaps
    t0 = time.perf_counter()                                # one call: seconds of host work would buy no precision
    h = community_overlaps(*b.F_csr(), b.K, delta, 1, everywhere)
    res[f"{tag}_host_route_s"] = time.perf_counter() - t0
    res[f"{tag}_arrays_equal"] = bool(all(np.array_equal(np.asarray(g[k]).view(np.uint8), np.asarray(h[k]).view(np.uint8))
                                          for k in ("ptr", "other", "shared", "size", "jaccard")))


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
    _work(b, coded, res, "amazon")
    for everywhere in (True, False):
        tag = f"amazon_zero_rows_{'everywhere' if everywhere else 'nowhere'}"
        g = _gpu(b, coded, res, tag, args.reps, everywhere)
        _host(b, coded, g, res, tag, everywhere)
    b.close()

    # com-amazon, synthetic F0 after 2 steps, K = 2000 and 9000
    for K in (2000, 9000):
        b = BigClam(sparse_rows=True)
        b.set_graph(rp, col).set_K(K).set_F_csr(*G.synthetic_F0_csr(n, K, seed=1234, density=0.05))
        for _ in range(2):
            b.backtrackingLineSearchs()
        _work(b, coded, res, f"K{K}")
        g = _gpu(b, coded, res, f"K{K}", args.reps)
        res[f"K{K}_jaccard_ge_half_pairs_nowhere"] = _jaccard_pairs(g, False)
        b.close()

    # planted, n = 10^6, K = 1000
    from bench_sample import _planted
    n, K = 1_000_000, 1000
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(*_planted(n, K, 0.15, 0.3, seed=3))
    _work(b, 0.1, res, "planted")
    g = _gpu(b, 0.1, res, "planted", args.reps)
    _host(b, 0.1, g, res, "planted", True)
    b.close()

    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_community_overlaps.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
