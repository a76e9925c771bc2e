"""The engine's size-dependent dispatch, restated for the large-batch tests: the constants of the CUDA sources, the GEMM
shape heuristics, and the seeded production-size graphs the cases run on (built once per process)."""
import functools

import numpy as np

from tf_gnn_samples_b200 import batching

# dispatch constants of the CUDA sources, restated
SMS = 132                    # RGNN_WAVE_SMS (csrc/common.cuh): persistent GEMM grid, one CTA per SM
SMALL_BATCH = SMS * 40       # seg_kernels.cu: below this many 128-column warps the half-warp kernels / split layer norm run
HEAVY_SEGMENT = 512          # RGNN_HEAVY_SEGMENT (csrc/plan.cuh): targets above it are reduced by several CTAs
GRU_SLAB = SMS * 128         # layers.cu: rows of one GRU-cell slab
TILE_M, TILE_K = 128, 32     # gemm_wgmma.cu: rows per tile, K per ring stage


def pick_bn(m_tiles, n_total, gz=1):
    """gemm_wgmma.cu pick_bn: the BN whose tiles take the fewest waves, weighted by the per-tile cost 96 + BN."""
    best, best_cost = 32, 1e30
    for bn in (128, 64, 32):
        waves = -(-(m_tiles * -(-n_total // bn) * gz) // SMS)
        cost = waves * (96.0 + bn)
        if cost < best_cost - 1e-9:
            best, best_cost = bn, cost
    return best


def ring_stages(bn):
    """gemm_wgmma.cu: stages of hi/lo A (128 rows) and B (BN rows) images of 128-byte rows in 227 KB, at most 4."""
    return min(4, (227 * 1024 - 1024 - 256) // (2 * 128 * 128 + 2 * bn * 128))


def gemm_shape(rows, n, k, k2=0, gz=1, row_counts=None):
    """BN, total tiles and K chunks of one launch_gemm_tc call (row_counts: the per-entry rows of BATCH_ROW_RANGES)."""
    bn = pick_bn(-(-rows // TILE_M), n, gz)
    counts = row_counts if row_counts is not None else [rows] * gz
    tiles = sum(-(-r // TILE_M) for r in counts) * -(-n // bn)
    return bn, tiles, -(-k // TILE_K) + -(-k2 // TILE_K)


# ------------------------------------------------------------------ graphs -----------------------------------------
def zipf_isolated_graph(num_nodes, edges_per_type, num_types, isolated, seed):
    """Uniform sources, Zipf(1)-skewed targets drawn from all but `isolated` nodes: hubs far above the heavy threshold and
    targets with no incoming edge at all."""
    rng = np.random.default_rng(seed)
    receivers = rng.permutation(num_nodes)[: num_nodes - isolated]
    p = 1.0 / np.arange(1, receivers.size + 1)
    p /= p.sum()
    adj = []
    for _ in range(num_types):
        src = rng.integers(0, num_nodes, size=edges_per_type)
        tgt = receivers[rng.choice(receivers.size, size=edges_per_type, p=p)]
        adj.append(np.stack([src, tgt], axis=1).astype(np.int32))
    indeg = np.stack([np.bincount(a[:, 1], minlength=num_nodes) for a in adj]).astype(np.float32)
    return adj, indeg


@functools.lru_cache(maxsize=4)
def graph(key):
    """(adjacency lists, in-degrees [L, V], V) of a graph key."""
    kind = key[0]
    if kind == "ppi":                     # ("ppi", V, links, seed, zipf): fwd / self-loop / bkwd types
        b = batching.ppi_like_batch(num_nodes=key[1], num_links=key[2], seed=key[3], zipf_targets=key[4])
    elif kind == "qm9":                   # ("qm9", molecules, seed): 4 bond types, ~18 atoms per molecule
        b = batching.qm9_like_batch(key[1], seed=key[2])
    else:                                 # ("zipf", V, edges per type, L, isolated, seed)
        adj, indeg = zipf_isolated_graph(*key[1:])
        return adj, indeg, key[1]
    return b.adjacency_lists, b.type_to_num_incoming_edges, b.num_nodes


def in_degrees(adj, V):
    return np.bincount(np.concatenate([a[:, 1] for a in adj]), minlength=V)


def segment_sizes(adj, V, by):
    """Edges per segment of the plan GraphPlan.regrouped(by) builds ('target': the plan itself; 'source_type' is also the
    reverse index of the edge-aggregate backward)."""
    L = len(adj)
    if by == "target":
        ids, n = np.concatenate([a[:, 1] for a in adj]), V
    elif by == "source":
        ids, n = np.concatenate([a[:, 0] for a in adj]), V
    elif by == "source_type":
        ids, n = np.concatenate([a[:, 0].astype(np.int64) * L + l for l, a in enumerate(adj)]), V * L
    elif by == "target_type":
        ids, n = np.concatenate([a[:, 1].astype(np.int64) * L + l for l, a in enumerate(adj)]), V * L
    else:
        raise ValueError(by)
    return np.bincount(ids, minlength=n)


def runs_crossing_chunks(adj, V):
    """Targets whose sorted (target, type) run continues across a 32-edge chunk of the edge kernel's loop."""
    tgt = np.concatenate([a[:, 1] for a in adj])
    typ = np.concatenate([np.full(a.shape[0], l) for l, a in enumerate(adj)])
    order = np.lexsort((typ, tgt))
    t, y = tgt[order], typ[order]
    seg = np.concatenate([[0], np.cumsum(np.bincount(tgt, minlength=V))])
    pos = np.arange(t.size) - seg[t]
    cont = np.r_[False, (t[1:] == t[:-1]) & (y[1:] == y[:-1])]
    return np.unique(t[cont & (pos % 32 == 0)]).size


def pair_rows_per_type(adj):
    """Rows of the compact (source, type) transform table per type (plan.cu pair table)."""
    return [np.unique(a[:, 0]).size for a in adj]


PPI6K_DENSE = ("ppi", 6000, 120000, 41, False)      # M = 246,000: ~41 incoming edges per target over 3 types
PPI6K = ("ppi", 6000, 18000, 44, False)             # M = 42,000, every node has its self loop
PPI6K_ZIPF = ("ppi", 6000, 24000, 45, True)         # hubs with thousands of incoming edges
QM9_20K = ("qm9", 1120, 7)                          # ~20,000 atoms
ZIPF6K = ("zipf", 6000, 12000, 3, 300, 46)          # 36,000 edges, >= 300 targets without an incoming edge
