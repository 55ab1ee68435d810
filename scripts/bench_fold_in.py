"""Fold-in on com-amazon: 1 % of the nodes are held out (dropped with their edges), F is fitted on the rest at K = 200
(initNeighborComF + SGDFindC), and the held-out nodes are folded in through their true neighbour lists.  Also timed:
every node's own neighbour list folded into a fit of the whole graph at K = 200 and at K = 2000 (SGDFindC capped at
--max-outer calls there), and the host route, a loop of oracle steps on the graph with the node appended, for a few
nodes.  Times are host clocks around synchronous calls, the best of --reps after a warm-up; the card's name and power
limit are read in the same run.  One quality figure is printed, not asserted: the mean p over the held-out nodes' true
edges against the mean p over random pairs of a held-out node and a fitted node.

    python scripts/bench_fold_in.py [--out DIR] [--reps N] [--host-nodes N]

Prints one JSON line (and writes it to DIR/bench_fold_in.json when --out is given)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
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
    return min(ts)


def _hold_out(rp, col, frac, seed):
    """(rp, col) of the kept nodes (relabelled), the held-out ids and their lists in the new labels."""
    n = len(rp) - 1
    rng = np.random.default_rng(seed)
    held = np.sort(rng.choice(n, max(1, int(frac * n)), replace=False))
    keep = np.ones(n, dtype=bool)
    keep[held] = False
    new = np.cumsum(keep) - 1
    u = np.repeat(np.arange(n), np.diff(rp))
    e = keep[u] & keep[col]
    nk = int(keep.sum())
    rpk = np.zeros(nk + 1, dtype=np.int64)
    rpk[1:] = np.cumsum(np.bincount(new[u[e]], minlength=nk))
    lists = [new[col[rp[h]:rp[h + 1]][keep[col[rp[h]:rp[h + 1]]]]] for h in held]
    qrp = np.zeros(len(held) + 1, dtype=np.int64)
    qrp[1:] = np.cumsum([len(x) for x in lists])
    return rpk, new[col[e]].astype(np.int32), qrp, np.concatenate(lists).astype(np.int32)


def _x(ip, ix, vl, F, us, vs):
    """x = row us[i] of (ip, ix, vl) dotted with F[vs[i]] (scipy)."""
    import scipy.sparse as S
    R = S.csr_matrix((vl, ix, ip), shape=(len(ip) - 1, F.shape[1]))
    return np.asarray(R[us].multiply(F[vs]).sum(axis=1)).ravel()


def _oracle_rows(O, rp, col, F, sumF, K, lists, max_iter, rel_tol):
    """The host route: the definition as a loop of oracle steps on G + u, one node at a time."""
    n = F.shape[0]
    params = O.make_params(K)
    mask = np.zeros(n + 1, dtype=np.uint8)
    mask[n] = 1
    for lst in lists:
        rp2 = np.concatenate([rp, [rp[-1] + len(lst)]]).astype(np.int64)
        col2 = np.concatenate([col, lst]).astype(np.int32)
        Fx = np.vstack([F, np.zeros((1, K))])
        lprev = None
        for it in range(max_iter + 1):
            r = O.step(rp2, col2, Fx, sumF + Fx[n], params, node_mask=mask, want_pre=True)
            lu = float(r.llh_u[n])
            if (it > 0 and abs(1.0 - lu / lprev) < rel_tol) or it == max_iter or r.accepted[n] < 0:
                break
            Fx[n] = r.F[n]
            lprev = lu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-nodes", type=int, default=3, help="nodes of the host route")
    ap.add_argument("--max-outer", type=int, default=30, help="SGDFindC calls of the K = 2000 fit")
    args = ap.parse_args()
    from bigclam_apachespark_b200 import BigClam, graphs as G
    from oracle import oracle as O

    rp, col, _ = G.load_npz_graph("com-amazon")
    n = len(rp) - 1
    res = {"card": _card(), "graph": "com-amazon", "n": n}
    # held-out nodes, K = 200
    rpk, colk, qrp, qcol = _hold_out(rp, col, 0.01, seed=1)
    b = BigClam(sparse_rows=True)
    b.set_graph(rpk, colk)
    b.initNeighborComF(200)
    t0 = time.perf_counter()
    res["heldout_fit_llh"] = b.SGDFindC()
    res["heldout_fit_s"] = time.perf_counter() - t0
    q = len(qrp) - 1
    res["heldout_nodes"] = q
    res["heldout_fold_in_s"] = _best(lambda: b.fold_in(qrp, qcol), args.reps)
    ip, ix, vl, llh, iters = b.fold_in(qrp, qcol)
    res["heldout_iters_mean"] = float(iters.mean())
    res["heldout_nnz_per_row"] = float(ip[-1] / q)
    Fk = b.F
    us = np.repeat(np.arange(q), np.diff(qrp))
    rng = np.random.default_rng(2)
    ur = rng.integers(0, q, len(us))
    vr = rng.integers(0, len(rpk) - 1, len(us))
    maxp = b.MAX_P_
    p_true = 1.0 - np.clip(np.exp(-_x(ip, ix, vl, Fk, us, qcol)), b.MIN_P_, maxp)
    p_rand = 1.0 - np.clip(np.exp(-_x(ip, ix, vl, Fk, ur, vr)), b.MIN_P_, maxp)
    res["heldout_mean_p_true_edges"] = float(p_true.mean())
    res["heldout_mean_p_random_pairs"] = float(p_rand.mean())
    # the host route for a few held-out nodes
    lists = [qcol[qrp[i]:qrp[i + 1]] for i in range(min(q, args.host_nodes))]
    t0 = time.perf_counter()
    _oracle_rows(O, rpk, colk, Fk, b.sumF, 200, lists, 100, 1e-4)
    th = time.perf_counter() - t0
    res["host_route_nodes"] = len(lists)
    res["host_route_s"] = th
    res["host_route_s_per_node"] = th / len(lists)
    b.close()
    # every node's own list folded into a fit of the whole graph
    for K in (200, 2000):
        b = BigClam(sparse_rows=True)
        b.set_graph(rp, col)
        b.initNeighborComF(K)
        b.SGDFindC(max_outer=0 if K == 200 else args.max_outer)
        res[f"all_nodes_K{K}_s"] = _best(lambda: b.fold_in(rp, col), args.reps)
        res[f"all_nodes_K{K}_nodes_per_s"] = n / res[f"all_nodes_K{K}_s"]
        b.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_fold_in.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
