"""NumPy model of the sparse-row tile path's cut and capacities (csrc/bigclam_capi.cu rebuild_sparse_lists / retile,
csrc/bigclam_tile.cuh TlWarp::run).  It predicts, per tile of a step kernel, whether the tile runs on the tile path or
falls back to the general path, and which check sends it there.  It predicts only: the oracle stays the reference for
every value.  The capacities are read from the kernel header's #define defaults, so a retune moves the tests with it.

The six checks of TlWarp::run, in the order the kernel makes them:
  stage   neighbour-row chunks total_e <= STAGE16, own-row chunks total_u <= OWN16, neighbour entries T <= EROW
  slots   touched components, summed over the tile's nodes: total_slots <= SLOTS
  act     (line search only) active components (fu_c > 0 or grad_c > 0), plus one padding slot: A <= ACT - 1
  ent     (only if a node is line-searched) entries of the searched nodes' neighbours on that node's active components,
          plus one padding entry: TE <= ENT - 1
"""
import os
import re

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "bigclam_apachespark_b200", "csrc")

MIN_P, MAX_P, MIN_F, MAX_F = 0.0001, 0.9999, 0.0, 1000.0
ALPHA = 0.05
STEPS = np.array([0.1 ** j for j in range(16)])         # candidates 1, 0.1, ..., 1e-15 (MaxInter = 15)
WIDE_LD = 1024                                          # above: wide rows, no tiles


def _header_defaults():
    with open(os.path.join(CSRC, "bigclam_tile.cuh")) as fh:
        src = fh.read()
    d = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define BIGCLAM_TL_(\w+) (\d+)\s*$", src, re.M)}
    for name in ("MaxNodes", "MaxEdges"):
        d[name] = int(re.search(r"constexpr int kTl%s = (\d+);" % name, src).group(1))
    with open(os.path.join(CSRC, "bigclam_sparse.cuh")) as fh:
        d["HubSeg"] = int(re.search(r"constexpr int kSpHubSeg = (\d+);", fh.read()).group(1))
    return d


_D = _header_defaults()
STAGE16, OWN16, SLOTS, ACT, ENT, EROW = (_D[k] for k in ("STAGE16", "OWN16", "SLOTS", "ACT", "ENT", "EROW"))
MAX_NODES, MAX_EDGES = _D["MaxNodes"], _D["MaxEdges"]
HUB_DEG_MIN = 2 * _D["HubSeg"]          # split hubs: deg >= max(2 * kSpHubSeg, share / 8)

# the largest value of each quantity that still fits (the two padding slots / entries are taken off)
LIMITS = {"stage_e": STAGE16, "stage_u": OWN16, "erow": EROW, "slots": SLOTS, "act": ACT - 1, "ent": ENT - 1}
CHECK_ORDER = ("stage_e", "stage_u", "erow", "slots", "act", "ent")
QUANTITY = {"stage_e": "total_e", "stage_u": "total_u", "erow": "T", "slots": "total_slots", "act": "A", "ent": "TE"}


def sp_words(c):
    """8-byte words of a sparse row block of c entries (bigclam_sparse.cuh sp_words)."""
    c = np.asarray(c, dtype=np.int64)
    return ((c + 1) & ~1) + ((c + 7) & ~7) // 4


def chunks(c):
    """16-byte chunks a row of c entries takes in the staging buffers."""
    return sp_words(c) >> 1


# ---------------------------------------------------------------------------------------------------------------
# the cut
def cut(rowptr, tile_edges=MAX_EDGES, tile_nodes=MAX_NODES, ld=None, hub_deg=None):
    """Processing order (degree descending, stable by id), split hubs, general-path nodes and tiles.
    Returns dict(order, n_hubs, n_gen, tiles = [array of node ids per tile])."""
    deg = np.diff(np.asarray(rowptr, dtype=np.int64))
    order = np.argsort(-deg, kind="stable")
    d = deg[order]
    hub = HUB_DEG_MIN if hub_deg is None else hub_deg
    nh = 0
    while nh < len(d) and d[nh] >= hub:
        nh += 1
    budget = 0 if (ld is not None and ld > WIDE_LD) else tile_edges
    pos = nh
    while pos < len(d) and (budget <= 0 or d[pos] > budget):
        pos += 1
    n_gen = pos - nh
    tiles = []
    while pos < len(d):
        p0, nn, ne = pos, 0, 0
        while pos < len(d) and nn < tile_nodes and ne + d[pos] <= budget:
            ne += d[pos]
            nn += 1
            pos += 1
        tiles.append(order[p0:pos])
    return dict(order=order, n_hubs=nh, n_gen=n_gen, tiles=tiles)


def retile_budget(rowptr, F, k):
    """The tile budget retile() picks when F is set (BIGCLAM_TILE_EDGES unset): (tile_edges, tile_nodes)."""
    n = len(rowptr) - 1
    cnt = (F != 0).sum(axis=1)
    nn = float(max(1, n))
    avg_cnt = max(1.0, float(cnt.sum()) / nn)
    avg16 = max(1.0, float(sp_words(cnt).sum()) / 2.0 / nn)
    nodes = max(0, min(MAX_NODES, int(OWN16 / (1.15 * avg16))))
    rows = min(STAGE16 / (1.1 * avg16), SLOTS / (1.1 * avg_cnt) - nodes)
    budget = max(0, min(MAX_EDGES, int(rows)))
    if budget < 6 or nodes < 2:
        budget = 0
    if budget == MAX_EDGES and nodes == MAX_NODES:
        return MAX_EDGES, MAX_NODES
    return budget, max(1, nodes)


# ---------------------------------------------------------------------------------------------------------------
# per node: gradient, active components, Armijo margins
def _edge_term(x):
    p = np.minimum(np.maximum(np.exp(-x), MIN_P), MAX_P)
    return np.log(1.0 - p) + x, p


def node_pre(rowptr, col, F, sumF, u):
    """(grad, llh_u, FV) of node u as the oracle defines them: grad = sum_v fv / (1 - p) - (sumF - fu)."""
    nb = col[rowptr[u]:rowptr[u + 1]]
    fu = F[u]
    FV = F[nb]
    t, p = _edge_term(FV @ fu)
    grad = (FV * (1.0 / (1.0 - p))[:, None]).sum(axis=0) - sumF + fu
    llh_u = t.sum() - fu @ sumF + fu @ fu
    return grad, llh_u, FV


def margins(rowptr, col, F, sumF, u):
    """Armijo margins llh'(s_j) - (llh_u + alpha s_j |g|^2) of node u's 16 candidates, and a rounding scale."""
    grad, llh_u, FV = node_pre(rowptr, col, F, sumF, u)
    fu = F[u]
    out = np.empty(len(STEPS))
    for j, s in enumerate(STEPS):
        nf = np.minimum(np.maximum(fu + s * grad, MIN_F), MAX_F)
        t, _ = _edge_term(FV @ nf)
        out[j] = t.sum() - nf @ (sumF - fu + nf) + nf @ nf - (llh_u + ALPHA * s * (grad @ grad))
    return out, max(abs(llh_u), 1.0)


class Ambiguous(AssertionError):
    """A prediction that would hinge on rounding: the construction must keep clear of it."""


def tile_quantities(rowptr, col, F, sumF, nodes, searched):
    """The six quantities of one tile.  `searched`: bool per node of the tile, whether it is line-searched."""
    nodes = np.asarray(nodes)
    cnt = (F != 0).sum(axis=1)
    q = dict(total_e=0, total_u=0, T=0, total_slots=0, A=0, TE=0)
    for i, u in enumerate(nodes):
        nb = col[rowptr[u]:rowptr[u + 1]]
        q["total_e"] += int(chunks(cnt[nb]).sum())
        q["total_u"] += int(chunks(cnt[u]))
        q["T"] += int(cnt[nb].sum())
        touched = F[u] != 0
        for v in nb:
            touched |= F[v] != 0
        q["total_slots"] += int(touched.sum())
        grad, _, FV = node_pre(rowptr, col, F, sumF, u)
        zero = touched & (F[u] == 0)
        scale = np.abs(FV).sum(axis=0) * (1.0 / (1.0 - MAX_P)) + np.abs(sumF) + 1.0
        if (zero & (np.abs(grad) <= 1e-9 * scale)).any():
            raise Ambiguous(f"node {u}: a touched zero component has a gradient at rounding level")
        active = touched & ((F[u] > 0) | (grad > 0))
        q["A"] += int(active.sum())
        if searched[i]:
            q["TE"] += int(sum(int(((F[v] != 0) & active).sum()) for v in nb))
    return q


def first_failure(q):
    """None if the tile runs on the tile path, else the first check that sends it to the general path."""
    if q["total_e"] > LIMITS["stage_e"]:
        return "stage_e"
    if q["total_u"] > LIMITS["stage_u"]:
        return "stage_u"
    if q["T"] > LIMITS["erow"]:
        return "erow"
    if q["total_slots"] > LIMITS["slots"]:
        return "slots"
    if q["A"] > LIMITS["act"]:
        return "act"
    if q["TE"] > LIMITS["ent"]:
        return "ent"
    return None


def predict_kernel(rowptr, col, F, sumF, tiles, exhaustive, node_mask=None):
    """One step kernel (with the line search): per tile (quantities, first failing check or None).  With the line-search bounds on, a node is
    surely searched when one of its candidates passes the Armijo test clearly (a sound bound cannot exclude it); a node
    without such a candidate may or may not be: when that decides the TE check, Ambiguous is raised."""
    rowptr = np.asarray(rowptr)
    deg = np.diff(rowptr)
    out = []
    for nodes in tiles:
        want = np.array([deg[u] > 0 and (node_mask is None or node_mask[u] != 0) for u in nodes], dtype=bool)
        if exhaustive:
            sure = want
        else:
            sure = np.zeros_like(want)
            for i, u in enumerate(nodes):
                if want[i]:
                    m, sc = margins(rowptr, col, F, sumF, u)
                    sure[i] = (m > 1e-7 * sc).any()
        q = tile_quantities(rowptr, col, F, sumF, nodes, want)
        fail = first_failure(q)
        if not (sure == want).all():
            qmin = tile_quantities(rowptr, col, F, sumF, nodes, sure)
            if first_failure(qmin) != fail:
                raise Ambiguous(f"tile {list(nodes)}: the TE check depends on which nodes the bounds exclude")
        out.append((q, fail))
    return out


def predict_counts(per_tile):
    done = sum(1 for _, f in per_tile if f is None)
    return done, len(per_tile) - done
