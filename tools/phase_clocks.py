"""Phase profile of the tile path on the bench workload (com-amazon, K = 200, synthetic F0): where the warps' cycles go.
    tools/build_variant.sh v_pc -DBIGCLAM_TL_PHASE_CLOCKS      (a build with clock64() stamps in TlWarp::run)
    python tools/phase_clocks.py v_pc [w_pc ...]                 (on a GPU; libraries tools/ab/lib_<v>.so, one process)
    tools/build_variant.sh v_pc4 -DBIGCLAM_TL_PHASE_CLOCKS -DBIGCLAM_TL_WARPS=4   (diagnostic: one warp per
                                 sub-partition, so a phase's cycles are its latency alone; the ratio to the 20-warp
                                 profile tells latency chains from issue-bound phases)
Warm-up and retile as bench.py does them, then 50 timed steps.  For each library: per bucket (hub items, general-path
nodes, tiles of nn nodes) the items, their share of all item cycles, and each phase's share of the bucket's cycles.  The
stamps, one global add each per phase and tile, slow the kernel down: this explains where the time goes, it is not a
timing.  Stamps 9 and 10 (H2.fold, H2.cand) sit inside the bounds' branch: with the bounds off (BIGCLAM_LS_PRUNE=0)
their time is counted in H2.sv.  DEV TOOL, never ships."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bigclam_apachespark_b200 import _lib, graphs as G  # noqa: E402
from bigclam_apachespark_b200.driver import BigClam  # noqa: E402

K, WARMUP, STEPS = 200, 5, 50
BUCKETS, SLOTS = 10, 18                  # kTlPcBuckets, kTlPcSlots (bigclam_tile.cuh)
WHOLE, ITEMS = SLOTS - 2, SLOTS - 1      # kTlPcWhole, kTlPcItems
# H and H2 in sub-phases: H = grad (the loop over slots), red (group reductions, active counts), walk (Dp/En per
# edge); H2 = lnthr (per-edge lnthr/Lp), fold (per-node Dp/En/viol), cand (candidate walk and bound), sv (svbits/n_sl)
PHASES = ["A", "B,C1", "E,C2", "C3,D", "G", "H.grad", "H.red", "H.walk", "H2.lnth", "H2.fold", "H2.cand", "H2.sv",
          "compact", "I", "J,K", "L"]


def profile(name):
    _lib._lib = None
    _lib.LIB_PATH = os.path.join(ROOT, "tools", "ab", f"lib_{name}.so")
    lib = _lib.load()
    fn = lib.bigclam_phase_clocks
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.POINTER(C.c_ulonglong)]
    rp, col, _ = G.load_npz_graph("com-amazon")
    F0 = G.synthetic_F0(len(rp) - 1, K, seed=1234, density=0.05)
    b = BigClam(device=0, sparse_rows=True)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    b._run(4, 0.0, WARMUP)
    for _ in range(3):
        b.retile()
        b._run(4, 0.0, 2)
    out = (C.c_ulonglong * (BUCKETS * SLOTS))()
    assert fn(b._need(), out) == 0                       # counters from zero
    b._run(4, 0.0, STEPS)
    assert fn(b._need(), out) == 0
    b.close()
    return np.array(out[:], dtype=np.float64).reshape(BUCKETS, SLOTS)


def report(name, pc):
    total = pc[:, WHOLE].sum()
    print(f"== {name}: {total:.4g} warp cycles in items over {STEPS} steps")
    print(f"{'bucket':>8} {'items':>10} {'cyc/item':>9} {'share':>6} " + " ".join(f"{p:>7}" for p in PHASES) + "   (phase % of the bucket's cycles)")
    labels = ["hub", "general"] + [f"nn={n}" for n in range(1, 9)]
    for bk in range(BUCKETS):
        items, cyc = pc[bk, ITEMS], pc[bk, WHOLE]
        if items == 0:
            continue
        ph = " ".join(f"{100 * pc[bk, k] / cyc:7.1f}" for k in range(len(PHASES))) if bk >= 2 else ""
        print(f"{labels[bk]:>8} {int(items):>10} {cyc / items:9.0f} {100 * cyc / total:5.1f}% {ph}")
    tiles = pc[2:].sum(axis=0)
    print(f"{'tiles':>8} {int(tiles[ITEMS]):>10} {tiles[WHOLE] / tiles[ITEMS]:9.0f} {100 * tiles[WHOLE] / total:5.1f}% "
          + " ".join(f"{100 * tiles[k] / tiles[WHOLE]:7.1f}" for k in range(len(PHASES))))
    print(f"{'cyc/tile':>8} {'':>10} {'':>9} {'':>6} " + " ".join(f"{tiles[k] / tiles[ITEMS]:7.0f}" for k in range(len(PHASES))))


if __name__ == "__main__":
    for v in sys.argv[1:]:
        report(v, profile(v))
