"""Building blocks of the hot path exported on their own (include/rgnn.h 'building blocks'):
the tensor-core Dense, the segment aggregation of utils.get_aggregation_function, and layer norm."""
from typing import Optional

import torch

from .engine import GraphPlan, RgnnError, RGNN_E_INVALID, as_f32, check, current_stream_ptr, load_library, output_rows, workspace
from .utils import get_activation, get_aggregation_function
from .utils import AGG_MAX, AGG_MEAN, AGG_SQRT_N, AGG_SUM
from .utils import (ACT_ELU, ACT_GELU, ACT_LEAKY_RELU, ACT_LINEAR, ACT_RELU, ACT_SELU, ACT_TANH)

# torch spellings of utils/utils.py:36-58 for the differentiable paths
_TORCH_ACT = {
    ACT_LINEAR: lambda t: t, ACT_TANH: torch.tanh, ACT_RELU: torch.relu,
    ACT_LEAKY_RELU: lambda t: torch.nn.functional.leaky_relu(t, 0.2), ACT_ELU: torch.nn.functional.elu,
    ACT_SELU: torch.selu, ACT_GELU: lambda t: torch.nn.functional.gelu(t),
}


def _dense_raw(x, kernel, b, act_code):
    out = torch.empty((x.shape[0], kernel.shape[1]), dtype=torch.float32, device=x.device)
    lib = load_library()
    with torch.cuda.device(x.device):
        ws = workspace(x.device, lib.rgnn_dense_workspace_bytes(x.shape[0], x.shape[1], kernel.shape[1]))
        check(lib.rgnn_dense_forward(x.data_ptr(), x.shape[0], x.shape[1], kernel.data_ptr(), kernel.shape[1],
                                     b.data_ptr() if b is not None else None, act_code,
                                     out.data_ptr(), ws.data_ptr(), ws.numel(), current_stream_ptr(x.device)))
    return out


def dense_backward(x: torch.Tensor, kernel: torch.Tensor, grad_out: torch.Tensor, need_x: bool = True,
                   need_kernel: bool = True):
    """Gradients of y = x @ kernel: (grad_out @ kernel^T, x^T @ grad_out) through rgnn_dense_backward
    (wgmma 3xTF32; the x^T contraction is split-K over the rows, deterministic)."""
    x, kernel, g = as_f32(x, "x"), as_f32(kernel, "kernel"), as_f32(grad_out, "grad_out")
    gx = torch.empty_like(x) if need_x else None
    gk = torch.empty_like(kernel) if need_kernel else None
    lib = load_library()
    with torch.cuda.device(x.device):
        ws = workspace(x.device, lib.rgnn_dense_workspace_bytes(x.shape[0], x.shape[1], kernel.shape[1]))
        check(lib.rgnn_dense_backward(x.data_ptr(), x.shape[0], x.shape[1], kernel.data_ptr(), kernel.shape[1],
                                      g.data_ptr(), gx.data_ptr() if need_x else None,
                                      gk.data_ptr() if need_kernel else None, ws.data_ptr(), ws.numel(),
                                      current_stream_ptr(x.device)))
    return gx, gk


class _Linear(torch.autograd.Function):
    """x @ kernel with both gradients on the engine's GEMMs."""

    @staticmethod
    def forward(ctx, x, kernel):
        ctx.save_for_backward(x, kernel)
        return _dense_raw(x, kernel, None, ACT_LINEAR)

    @staticmethod
    def backward(ctx, grad_out):
        x, kernel = ctx.saved_tensors
        gx, gk = dense_backward(x, kernel, grad_out.contiguous(), ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return gx, gk


def dense(x: torch.Tensor, kernel: torch.Tensor, bias: Optional[torch.Tensor] = None,
          activation: Optional[str] = None) -> torch.Tensor:
    """act(x @ kernel + bias): tf.keras.layers.Dense with the Keras [in, out] kernel (SURVEY.md A.1),
    fp32-accurate on the tensor cores (wgmma 3xTF32).  Under autograd the contraction and both of its
    gradients run on the engine (bias / activation are then applied by torch so that autograd can chain them)."""
    x, kernel = as_f32(x, "x"), as_f32(kernel, "kernel")
    if x.dim() != 2 or kernel.dim() != 2 or x.shape[1] != kernel.shape[0]:
        raise RgnnError(RGNN_E_INVALID, "dense: shapes %s x %s do not contract" % (tuple(x.shape), tuple(kernel.shape)))
    b = as_f32(bias, "bias") if bias is not None else None
    act_code = get_activation(activation)
    needs_grad = torch.is_grad_enabled() and (x.requires_grad or kernel.requires_grad or (b is not None and b.requires_grad))
    if not needs_grad:
        return _dense_raw(x, kernel, b, act_code)
    if x.shape[1] % 4 or kernel.shape[1] % 4:
        raise RgnnError(RGNN_E_INVALID, "dense: gradients need input / output widths that are multiples of 4")
    y = _Linear.apply(x, kernel)
    if b is not None:
        y = y + b
    return _TORCH_ACT[act_code](y)


def _segment_raw(plan: GraphPlan, data: torch.Tensor, agg_code: int) -> torch.Tensor:
    out = output_rows(plan, data.shape[1], data.device)
    if data.shape[0] == 0:            # no messages: an empty tensor has no device pointer; the kernel never dereferences it
        data = torch.zeros((1, data.shape[1]), dtype=torch.float32, device=data.device)
    with torch.cuda.device(data.device):
        check(load_library().rgnn_segment_aggregate(plan.handle, data.data_ptr(), data.shape[1], agg_code,
                                                    out.data_ptr(), current_stream_ptr(data.device)))
    return out


class _SegmentAggregate(torch.autograd.Function):
    """tf.unsorted_segment_<agg> with TF's gradients: sum -> gather; mean / sqrt_n -> gather of grad / n, grad / sqrt(n);
    max -> the gradient goes to the entries equal to the maximum, split evenly among ties."""

    @staticmethod
    def forward(ctx, data, plan, agg_code):
        out = _segment_raw(plan, data, agg_code)
        ctx.plan, ctx.agg_code = plan, agg_code
        if agg_code == AGG_MAX:
            ctx.save_for_backward(data, out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        plan, agg = ctx.plan, ctx.agg_code
        tgt = plan.message_targets
        g = grad_out
        if agg == AGG_MEAN:
            g = g / plan.in_degree.clamp(min=1.0).unsqueeze(1)
        elif agg == AGG_SQRT_N:
            g = g / plan.in_degree.clamp(min=1.0).sqrt().unsqueeze(1)
        if agg != AGG_MAX:
            return g.index_select(0, tgt), None, None
        data, out = ctx.saved_tensors
        selected = (data == out.index_select(0, tgt)).float()
        ties = _segment_raw(plan, selected, AGG_SUM).clamp(min=1.0)
        return selected * (g / ties).index_select(0, tgt), None, None


def segment_aggregate(plan: GraphPlan, data: torch.Tensor, aggregation: str = "sum") -> torch.Tensor:
    """tf.unsorted_segment_<agg>(data, message_targets, num_nodes) for `data` [M, d] whose rows are in the
    type-major concatenation order of the adjacency lists the plan was built from (gnns/rgcn.py:108-112).
    Differentiable with respect to `data`."""
    data = as_f32(data, "data")
    if data.dim() != 2 or data.shape[0] != plan.num_edges:
        raise RgnnError(RGNN_E_INVALID, "segment_aggregate: data must be [M=%d, d], got %s" % (plan.num_edges, tuple(data.shape)))
    code = get_aggregation_function(aggregation)
    if torch.is_grad_enabled() and data.requires_grad:
        return _SegmentAggregate.apply(data, plan, code)
    return _segment_raw(plan, data, code)


class _EdgeAggregate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, plan, cnt, agg_code):
        V, L, d = table.shape
        out = output_rows(plan, d, table.device)
        with torch.cuda.device(table.device):
            check(load_library().rgnn_edge_aggregate_forward(plan.handle, table.data_ptr(), d,
                                                             cnt.data_ptr() if cnt is not None else None, agg_code,
                                                             out.data_ptr(), current_stream_ptr(table.device)))
        ctx.plan, ctx.cnt, ctx.agg_code, ctx.shape = plan, cnt, agg_code, (V, L, d)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        V, L, d = ctx.shape
        g = grad_out.contiguous()
        d_table = torch.empty((V, L, d), dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            check(load_library().rgnn_edge_aggregate_backward(ctx.plan.handle, g.data_ptr(), d,
                                                              ctx.cnt.data_ptr() if ctx.cnt is not None else None,
                                                              ctx.agg_code, d_table.data_ptr(), current_stream_ptr(g.device)))
        return d_table, None, None, None


def edge_aggregate(table: torch.Tensor, plan: GraphPlan, type_to_num_incoming_edges: Optional[torch.Tensor] = None,
                   aggregation: str = "sum") -> torch.Tensor:
    """out[v] = agg over incoming (u, v) of every type l of  table[u, l, :] / (c[l, v] + 1e-7)  (no scaling when the
    in-degrees are None): the fused edge stage on per-node transformed states ``table`` [V, L, d] -- no per-edge
    tensor is materialised in either direction.  Differentiable w.r.t. ``table`` for sum / mean / sqrt_n."""
    table = as_f32(table, "table")
    if table.dim() != 3 or table.shape[0] != plan.num_nodes or table.shape[1] != plan.num_edge_types:
        raise RgnnError(RGNN_E_INVALID, "edge_aggregate: table must be [V=%d, L=%d, d], got %s"
                        % (plan.num_nodes, plan.num_edge_types, tuple(table.shape)))
    cnt = as_f32(type_to_num_incoming_edges, "type_to_num_incoming_edges") if type_to_num_incoming_edges is not None else None
    return _EdgeAggregate.apply(table, plan, cnt, get_aggregation_function(aggregation))


class _Gather(torch.autograd.Function):
    """rows = table[index]; the backward segment-sums the per-edge gradients with the engine's deterministic kernel over
    a plan whose segments are the gathered rows (tf.nn.embedding_lookup's gradient is the same unsorted_segment_sum)."""

    @staticmethod
    def forward(ctx, table, index, back_plan):
        ctx.back_plan, ctx.rows = back_plan, table.shape[0]
        return table.index_select(0, index)

    @staticmethod
    def backward(ctx, grad_rows):
        g = _segment_raw(ctx.back_plan, grad_rows.contiguous(), AGG_SUM)
        return g[: ctx.rows], None, None


def gather_rows(x: torch.Tensor, plan: GraphPlan, side: str) -> torch.Tensor:
    """tf.nn.embedding_lookup(x, edge_sources | edge_targets) for all messages, type-major order (gnns/rgcn.py:88,93)."""
    x = as_f32(x, "x")
    if side == "source":
        return _Gather.apply(x, plan.message_sources, plan.regrouped("source"))
    if side == "target":
        return _Gather.apply(x, plan.message_targets, plan)
    raise RgnnError(RGNN_E_INVALID, "gather_rows: side must be 'source' or 'target'")


def gather_table_rows(table: torch.Tensor, plan: GraphPlan, side: str) -> torch.Tensor:
    """table [V, L, d] -> [M, d]: row (source | target of the message, its edge type)."""
    table = as_f32(table, "table")
    V, L, d = table.shape
    flat = table.reshape(V * L, d)
    if side == "source":
        return _Gather.apply(flat, plan.message_sources * L + plan.message_types, plan.regrouped("source_type"))
    if side == "target":
        return _Gather.apply(flat, plan.message_targets * L + plan.message_types, plan.regrouped("target_type"))
    raise RgnnError(RGNN_E_INVALID, "gather_table_rows: side must be 'source' or 'target'")


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor) -> torch.Tensor:
    """tf.contrib.layers.layer_norm defaults: last axis, biased variance, eps 1e-12 (SURVEY.md A.5)."""
    x, gamma, beta = as_f32(x, "x"), as_f32(gamma, "gamma"), as_f32(beta, "beta")
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(load_library().rgnn_layer_norm(x.data_ptr(), x.shape[0], x.shape[1], gamma.data_ptr(), beta.data_ptr(),
                                             out.data_ptr(), current_stream_ptr(x.device)))
    return out
