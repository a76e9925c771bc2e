"""Differentiable (training-mode) paths of the layer functions.

The inference paths of gnns/*.py are single fused library calls.  Under autograd (any input requiring a gradient)
sparse_rgcn_layer keeps its fused forward/backward kernels (rgnn_rgcn_backward); the other layers are composed here
from the engine's differentiable building blocks (ops.py) --

  * ops.dense            wgmma 3xTF32 GEMM, both gradients on the tensor cores (transposed-weight GEMM, split-K TN);
  * ops.edge_aggregate   the fused gather -> scale -> segment-reduce kernel on per-node tables [V, L, D] and its reverse
                         (segments = (source, type)) -- no per-edge tensor in either direction;
  * ops.segment_aggregate / ops.gather_rows / ops.gather_table_rows   for the layers whose messages are non-linear per
                         edge (FiLM, Edge-MLP, RGAT, target-conditioned RGIN): per-edge [M, D] tensors are materialised
                         like the reference does, gathers / scatters run on the engine's deterministic segment kernels;

-- with torch elementwise ops in between so autograd can chain them.  Same re-associations as the inference kernels
(transform per node first, then aggregate; DESIGN.md 3), same results as the reference op order up to fp32 rounding.
The reference obtains these gradients from TF autodiff (models/sparse_graph_model.py:253-260).
"""
from typing import Dict, List, Optional

import torch

from .. import ops
from ..engine import GraphPlan, RgnnError, RGNN_E_INVALID
from ..utils import AGG_MAX, get_activation, get_aggregation_function

_ACT = ops._TORCH_ACT


def requires_grad(*objs) -> bool:
    """True when autograd is recording and any tensor inside the (nested) containers requires a gradient."""
    if not torch.is_grad_enabled():
        return False

    def walk(o):
        if isinstance(o, torch.Tensor):
            return o.requires_grad
        if isinstance(o, dict):
            return any(walk(v) for v in o.values())
        if isinstance(o, (list, tuple)):
            return any(walk(v) for v in o)
        return False
    return any(walk(o) for o in objs)


def _check_restricted(plan: GraphPlan, num_timesteps: int):
    """A plan restricted to its first num_targets rows (one rank of a node-range partition) updates only those rows: the
    halo rows must be refreshed by the caller's exchange between steps, so -- like the C ABI -- only one timestep per call."""
    if getattr(plan, "num_targets", plan.num_nodes) < plan.num_nodes and int(num_timesteps) != 1:
        raise RgnnError(RGNN_E_INVALID, "a plan restricted to %d of %d target rows supports num_timesteps == 1 only"
                        % (plan.num_targets, plan.num_nodes))


def _layer_norm(x, gamma, beta):
    return torch.nn.functional.layer_norm(x, (x.shape[1],), gamma, beta, 1e-12)     # tf.contrib.layers.layer_norm (A.5)


def _message_scale(plan: GraphPlan, cnt: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """[M, 1]: 1 / (c[type, target] + 1e-7) per message (gnns/rgcn.py:100-104); constant w.r.t. autograd."""
    if cnt is None:
        return None
    return (1.0 / (cnt[plan.message_types, plan.message_targets] + 1e-7)).unsqueeze(1)


def _aggregate_table(table, plan, cnt, aggregation: str):
    """agg over incoming messages of s * table[source, type]: fused kernel for sum / mean / sqrt_n, per-edge path for max."""
    if get_aggregation_function(aggregation) != AGG_MAX:
        return ops.edge_aggregate(table, plan, cnt, aggregation)
    rows = ops.gather_table_rows(table, plan, "source")
    scale = _message_scale(plan, cnt)
    return ops.segment_aggregate(plan, rows if scale is None else rows * scale, aggregation)


def _mlp(kernels: List[torch.Tensor], x, hidden_act):
    """utils/utils.py:77-126."""
    for k in kernels[:-1]:
        x = hidden_act(ops.dense(x, k))
    return ops.dense(x, kernels[-1])


def _per_type_mlp(mlps, x, plan: GraphPlan, hidden_act):
    """Rows of x are messages in type-major order: apply MLP_l to the block of type l."""
    off = plan.type_offsets
    outs = []
    for l, ks in enumerate(mlps):
        if off[l + 1] > off[l]:
            outs.append(_mlp(ks, x[off[l]:off[l + 1]], hidden_act))
    if not outs:
        return x.new_zeros((0, mlps[0][-1].shape[1]))
    return torch.cat(outs, dim=0)


# ---- gnns/rgcn.py:84-114 for the settings the fused backward does not cover (max aggregation / [h_u | h_v] messages) ----
def rgcn(h, plan, cnt, ws, act_code, aggregation, use_both, num_timesteps):
    _check_restricted(plan, num_timesteps)
    act = _ACT[act_code]
    L, d_out = plan.num_edge_types, ws[0].shape[1]
    cur = h
    for _ in range(int(num_timesteps)):
        d_in = cur.shape[1]
        table = ops.dense(cur, torch.cat([w[:d_in] for w in ws], dim=1)).view(-1, L, d_out)
        if not use_both:
            cur = act(_aggregate_table(table, plan, cnt, aggregation))
            continue
        q = ops.dense(cur, torch.cat([w[d_in:] for w in ws], dim=1)).view(-1, L, d_out)   # [h_u | h_v] W = h_u W_src + h_v W_tgt
        rows = ops.gather_table_rows(table, plan, "source") + ops.gather_table_rows(q, plan, "target")
        scale = _message_scale(plan, cnt)
        cur = act(ops.segment_aggregate(plan, rows if scale is None else rows * scale, aggregation))
    return cur


# ---- gnns/ggnn.py:71-93 ----
def ggnn(h, plan, ws, cell, cell_kind: str, act_code, aggregation, num_timesteps):
    _check_restricted(plan, num_timesteps)
    act = _ACT[act_code]
    L, d = plan.num_edge_types, h.shape[1]
    K, R, B = cell["kernel"], cell["recurrent_kernel"], cell["bias"]
    w_cat = torch.cat(list(ws), dim=1)
    cur = h
    for _ in range(int(num_timesteps)):
        m = _aggregate_table(ops.dense(cur, w_cat).view(-1, L, d), plan, None, aggregation)
        if cell_kind == "rnn":                                        # SimpleRNNCell: act(x W + b + h U)
            cur = act(ops.dense(m, K) + B + ops.dense(cur, R))
            continue
        xk = ops.dense(m, K) + B                                      # GRUCell, TF 1.13 defaults (gates z | r | h, hard_sigmoid)
        hr = ops.dense(cur, R[:, :2 * d])
        zr = torch.clamp(0.2 * (xk[:, :2 * d] + hr) + 0.5, 0.0, 1.0)
        z, r = zr[:, :d], zr[:, d:]
        hh = act(xk[:, 2 * d:] + ops.dense(r * cur, R[:, 2 * d:]))
        cur = z * cur + (1.0 - z) * hh
    return cur


# ---- gnns/rgat.py:83-138 ----
def rgat(h, plan, ws, att, num_heads: int, act_code, num_timesteps):
    _check_restricted(plan, num_timesteps)
    act = _ACT[act_code]
    L, V = plan.num_edge_types, plan.num_nodes
    D = ws[0].shape[1]
    dh = D // num_heads
    w_cat = torch.cat(list(ws), dim=1)
    a = torch.stack(list(att)).view(L, num_heads, 2 * dh)             # head k of type l: [k*2dh, (k+1)*2dh) (rgat.py:110-111)
    src_t = plan.message_sources * L + plan.message_types
    tgt_t = plan.message_targets * L + plan.message_types
    tgt = plan.message_targets
    cur = h
    for _ in range(int(num_timesteps)):
        table = ops.dense(cur, w_cat).view(V, L, D)
        t4 = table.view(V, L, num_heads, dh)
        s_src = (t4 * a[:, :, :dh].unsqueeze(0)).sum(-1).view(V * L, num_heads)       # <a_src, T[u, l, k]>
        s_tgt = (t4 * a[:, :, dh:].unsqueeze(0)).sum(-1).view(V * L, num_heads)
        e = torch.nn.functional.leaky_relu(s_src.index_select(0, src_t) + s_tgt.index_select(0, tgt_t), 0.2)   # [M, K]
        idx = tgt.unsqueeze(1).expand(-1, num_heads)
        mx = torch.full((V, num_heads), -3.4028234663852886e38, device=h.device).scatter_reduce(0, idx, e.detach(), "amax")
        ex = torch.exp(e - mx.index_select(0, tgt))
        den = torch.zeros((V, num_heads), device=h.device).index_add(0, tgt, ex)
        alpha = ex / den.index_select(0, tgt)                         # softmax over ALL incoming messages of the target, per head
        rows = ops.gather_table_rows(table, plan, "source").view(-1, num_heads, dh)
        cur = act(ops.segment_aggregate(plan, (alpha.unsqueeze(-1) * rows).reshape(-1, D), "sum"))
    return cur


# ---- gnns/gnn_film.py:85-120 ----
def film(h, plan, cnt, ws, fws, ln, act_code, aggregation, num_timesteps):
    _check_restricted(plan, num_timesteps)
    act = _ACT[act_code]
    L, V, D = plan.num_edge_types, plan.num_nodes, ws[0].shape[1]
    w_cat, f_cat = torch.cat(list(ws), dim=1), torch.cat(list(fws), dim=1)
    scale = _message_scale(plan, cnt)
    cur = h
    for t in range(int(num_timesteps)):
        msg = ops.gather_table_rows(ops.dense(cur, w_cat).view(V, L, D), plan, "source")
        if scale is not None:
            msg = msg * scale
        pm = ops.gather_table_rows(ops.dense(cur, f_cat).view(V, L, 2 * D), plan, "target")
        agg = ops.segment_aggregate(plan, act(pm[:, :D] * msg + pm[:, D:]), aggregation)     # activation inside the sum (:111-116)
        cur = _layer_norm(agg, ln[0][t], ln[1][t])
    return cur


# ---- gnns/gnn_edge_mlp.py:84-119 ----
def edge_mlp(h, plan, cnt, mlps, ln, act_code, aggregation, use_target: bool, num_timesteps):
    _check_restricted(plan, num_timesteps)
    act, elu = _ACT[act_code], torch.nn.functional.elu
    D = mlps[0][-1].shape[1]
    scale = _message_scale(plan, cnt)
    cur = h
    for t in range(int(num_timesteps)):
        x = ops.gather_rows(cur, plan, "source")
        if use_target:
            x = torch.cat([x, ops.gather_rows(cur, plan, "target")], dim=1)
        msg = _per_type_mlp(mlps, x, plan, elu)
        if scale is not None:
            msg = msg * scale
        agg = ops.segment_aggregate(plan, act(msg), aggregation)
        cur = _layer_norm(agg, ln[0][t], ln[1][t])
    return cur


# ---- gnns/rgin.py:103-139 ----
def rgin(h, plan, mlps, aggr_mlp, ln, act_code, aggregation, use_target: bool, num_timesteps):
    _check_restricted(plan, num_timesteps)
    act = _ACT[act_code]
    L, V = plan.num_edge_types, plan.num_nodes
    cur = h
    for t in range(int(num_timesteps)):
        if not use_target and mlps is not None:
            # the message depends on (source, type) only: evaluate the edge MLPs per node, aggregate with the fused kernel
            table = torch.stack([act(_mlp(ks, cur, act)) for ks in mlps], dim=1)
            new = _aggregate_table(table, plan, None, aggregation)
        elif not use_target:
            new = _aggregate_table(cur.unsqueeze(1).expand(V, L, cur.shape[1]).contiguous(), plan, None, aggregation)
        else:
            x = torch.cat([ops.gather_rows(cur, plan, "source"), ops.gather_rows(cur, plan, "target")], dim=1)
            if mlps is not None:
                x = act(_per_type_mlp(mlps, x, plan, act))
            new = ops.segment_aggregate(plan, x, aggregation)
        if aggr_mlp is not None:
            new = _mlp(aggr_mlp, new, act)
        new = act(new)
        cur = _layer_norm(new, ln[0][t], ln[1][t])
    return cur
