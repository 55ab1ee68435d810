"""initNeighborComF(K) two ways: the host route (bigclam_init_neighbor_com_F fills an n x K array, bigclam_set_F loads it)
against init_F (bigclam_init_F builds the rows on the device, straight into the context).  com-amazon at K = 200, 1000,
2000 and 9000 (the host route is skipped where its n x K doubles exceed 4 GiB) and email-enron at K = 9000, where
most columns are random padding.  Each time is a host clock around synchronous calls, the best of --reps after a
warm-up, on a context created beforehand (sparse rows).  Where both routes ran, their F rows and sumF are compared.  A
capped sweep_K on com-amazon is split into init time and solver time.  The card's name and power limit are read in the
same run.

    python scripts/bench_init.py [--out DIR] [--reps N] [--sweep-outer N]

Prints one JSON line (and writes it to DIR/bench_init.json when --out is given)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.dont_write_bytecode = True

HOST_LIMIT = 4 << 30


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


def _host_route(b, K):
    from bigclam_apachespark_b200 import _lib
    F0 = np.empty((b.n, K), dtype=np.float64)
    rc = _lib.load().bigclam_init_neighbor_com_F(b.n, b.rowptr.ctypes.data, b.col.ctypes.data, K, b.Sbc.ctypes.data, len(b.Sbc),
                                                 0, C.c_uint64(1234), F0.ctypes.data)
    assert rc == _lib.OK
    b.set_F(F0)


def case(name, K, reps):
    from bigclam_apachespark_b200 import BigClam, graphs as G
    rp, col, _ = G.load_npz_graph(name)
    b = BigClam(sparse_rows=True).set_graph(rp, col)
    b.conductanceLocalMin()
    b.set_K(K)
    out = {"graph": name, "n": b.n, "K": K, "seeds": int(min(K, len(b.Sbc))), "host_F0_bytes": b.n * K * 8}
    out["init_F_s"] = _best(lambda: b.init_F(K), reps)
    g_csr, g_sum = b.F_csr(), b.sumF
    out["nnz_F0"] = int(len(g_csr[1]))
    if b.n * K * 8 <= HOST_LIMIT:
        out["host_route_s"] = _best(lambda: _host_route(b, K), reps)
        h_csr, h_sum = b.F_csr(), b.sumF
        out["same"] = bool(all(np.array_equal(x, y) for x, y in zip(g_csr, h_csr)) and np.array_equal(g_sum, h_sum))
        out["speedup"] = out["host_route_s"] / out["init_F_s"]
    else:
        out["host_route_s"] = None                              # n x K doubles above HOST_LIMIT: not run
    b.close()
    return out


def sweep(max_outer, lo, hi, div):
    from bigclam_apachespark_b200 import BigClam, graphs as G
    rp, col, _ = G.load_npz_graph("com-amazon")
    b = BigClam(minCom=lo, maxCom=hi, divCom=div, sparse_rows=True).set_graph(rp, col)
    b.conductanceLocalMin()
    t = {"init_F": 0.0, "SGDFindC": 0.0}

    def timed(key, fn):
        def call(*a, **kw):
            t0 = time.perf_counter()
            r = fn(*a, **kw)
            t[key] += time.perf_counter() - t0
            return r
        return call

    b.init_F = timed("init_F", b.init_F)           # (set_K, i.e. the context of each K, is timed inside init_F)
    b.SGDFindC = timed("SGDFindC", b.SGDFindC)
    t0 = time.perf_counter()
    KforC, hist = b.sweep_K(max_outer=max_outer)
    total = time.perf_counter() - t0
    b.close()
    return {"graph": "com-amazon", "Kset": [k for k, _ in hist], "max_outer": max_outer, "KforC": KforC, "total_s": total,
            "init_F_s": t["init_F"], "SGDFindC_s": t["SGDFindC"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sweep-outer", type=int, default=3)
    args = ap.parse_args()
    res = {"card": _card(), "cases": []}
    for name, K in [("com-amazon", 200), ("com-amazon", 1000), ("com-amazon", 2000), ("com-amazon", 9000), ("email-enron", 9000)]:
        res["cases"].append(case(name, K, args.reps))
        print(json.dumps(res["cases"][-1]), file=sys.stderr, flush=True)
    res["sweep"] = sweep(args.sweep_outer, 1000, 3000, 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_init.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
