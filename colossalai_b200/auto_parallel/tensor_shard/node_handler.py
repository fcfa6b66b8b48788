"""Strategy generators: one handler per kind of fx node.

Parity: reference `colossalai/auto_parallel/tensor_shard/node_handler/*` (linear / matmul / embedding / layer-norm /
elementwise / reshape / softmax / placeholder / output handlers and their strategy generators).  The handlers here are
organised around *roles*: every mesh axis is given a role for the node (unused, split a batch dimension, split the
output features, split the contraction, ...) and the operand / result layouts, the partial sums and the gradient
synchronisation all follow from the roles, so 1-D and 2-D meshes need no separate code.

Any node without a handler gets the single always-valid strategy "everything replicated".
"""
from __future__ import annotations

import itertools
import math
import operator
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch
import torch.fx as fx
import torch.nn as nn
import torch.nn.functional as F

from ...device import DeviceMesh
from .sharding_strategy import (ShardingStrategy, Spec, StrategiesVector, enumerate_specs, replicated, shard_factor,
                                spec_str)

__all__ = ["HandlerContext", "generate_strategies", "node_shape", "tensor_operands", "reshape_dim_map",
           "RESHAPE_METHODS", "register_module_handler", "register_function_handler"]


@dataclass
class HandlerContext:
    gm: fx.GraphModule
    mesh: DeviceMesh
    peak_flops: float = 1.4e15          # order of magnitude of a dense bf16 tensor-core GPU (H100 SXM data sheet: 0.99e15)
    hbm_bw: float = 6.0e12              # measured copy bandwidth
    shard_inputs: bool = True           # placeholders may be batch-split
    train: bool = True

    @property
    def mesh_shape(self) -> Tuple[int, ...]:
        return tuple(self.mesh.shape)

    def mm_time(self, flops: float, factor: int) -> float:
        return (3.0 if self.train else 1.0) * flops / (self.peak_flops * factor)

    def mem_time(self, nbytes: float, factor: int) -> float:
        return (3.0 if self.train else 1.0) * nbytes / (self.hbm_bw * factor)


# ---------------------------------------------------------------------------------------------------------- helpers
def node_meta(n: fx.Node):
    tm = n.meta.get("tensor_meta")
    if isinstance(tm, tuple) and len(tm) == 2 and isinstance(tm[0], tuple) and isinstance(tm[1], torch.dtype):
        return tm
    return None


def node_shape(n: fx.Node) -> Optional[Tuple[int, ...]]:
    tm = node_meta(n)
    return None if tm is None else tm[0]


def node_bytes(n: fx.Node) -> float:
    tm = node_meta(n)
    if tm is None:
        return 0.0
    return float(math.prod(tm[0])) * torch.empty((), dtype=tm[1]).element_size()


def tensor_operands(n: fx.Node) -> List[fx.Node]:
    return [a for a in n.all_input_nodes if node_shape(a) is not None]


def _axes(mesh_shape: Sequence[int]) -> List[int]:
    return [a for a, s in enumerate(mesh_shape) if s > 1]


def _used_axes(spec: Optional[Spec]) -> Tuple[int, ...]:
    return tuple(a for a in (spec or ()) if a is not None)


def _replicated_strategy(node: fx.Node, ctx: HandlerContext, cost: float = 0.0) -> ShardingStrategy:
    shape = node_shape(node)
    return ShardingStrategy(
        "replicate", None if shape is None else replicated(len(shape)),
        {a.name: replicated(len(node_shape(a))) for a in tensor_operands(node)},
        compute_cost=cost, memory_cost=node_bytes(node))


def _aligned_operand_spec(out_spec: Spec, out_shape: Sequence[int], op_shape: Sequence[int]) -> Spec:
    """Layout of a (broadcastable) elementwise operand under `out_spec`: a dimension follows the output only when it
    has the same extent; broadcast (size-1 / missing) dimensions stay whole."""
    off = len(out_shape) - len(op_shape)
    return tuple(out_spec[off + d] if op_shape[d] == out_shape[off + d] and op_shape[d] > 1 else None
                 for d in range(len(op_shape)))


# ---------------------------------------------------------------------------------------------------------- handlers
def placeholder_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    shape = node_shape(node)
    if shape is None:
        return [ShardingStrategy("replicate", None)]
    out = [ShardingStrategy("replicate", replicated(len(shape)), memory_cost=node_bytes(node))]
    if ctx.shard_inputs and len(shape) > 0:
        for spec in enumerate_specs(shape, ctx.mesh_shape, allowed_dims=[0]):
            if _used_axes(spec):
                out.append(ShardingStrategy(f"split{spec_str(spec)}", spec,
                                            memory_cost=node_bytes(node) / shard_factor(spec, ctx.mesh_shape)))
    return out


def get_attr_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    shape = node_shape(node)
    return [ShardingStrategy("replicate", None if shape is None else replicated(len(shape)),
                             memory_cost=node_bytes(node))]


def output_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    return [ShardingStrategy("replicate", None, {a.name: replicated(len(node_shape(a))) for a in tensor_operands(node)})]


def elementwise_handler(node: fx.Node, ctx: HandlerContext, forbid_dims: Sequence[int] = ()) -> List[ShardingStrategy]:
    """Unary / broadcasting n-ary pointwise ops: the result may take any layout; operands follow it."""
    shape = node_shape(node)
    ops = tensor_operands(node)
    if shape is None or not ops:
        return [_replicated_strategy(node, ctx)]
    nd = len(shape)
    bad = {d % nd for d in forbid_dims} if nd else set()
    allowed = [d for d in range(nd) if d not in bad]
    nbytes = node_bytes(node)
    out = []
    for spec in enumerate_specs(shape, ctx.mesh_shape, allowed_dims=allowed):
        f = shard_factor(spec, ctx.mesh_shape)
        ins, bwd, comm = {}, {}, 0.0
        for a in ops:
            ashape = node_shape(a)
            if len(ashape) > nd:
                ins = None
                break
            aspec = _aligned_operand_spec(spec, shape, ashape)
            ins[a.name] = aspec
            missing = tuple(x for x in _used_axes(spec) if x not in _used_axes(aspec))
            if missing and ctx.train:
                bwd[a.name] = missing
                comm += sum(ctx.mesh.all_reduce_cost(node_bytes(a), x) for x in missing)
        if ins is None:
            continue
        out.append(ShardingStrategy(f"pointwise{spec_str(spec)}", spec, ins, compute_cost=ctx.mem_time(2 * nbytes, f),
                                    comm_cost=comm, memory_cost=nbytes / f, bwd_reduce_inputs=bwd))
    return out or [_replicated_strategy(node, ctx)]


def softmax_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    dim = node.kwargs.get("dim", node.args[1] if len(node.args) > 1 else -1)
    if node.op == "call_module":
        dim = getattr(ctx.gm.get_submodule(node.target), "dim", -1)
    return elementwise_handler(node, ctx, forbid_dims=[-1 if dim is None else dim])


def reduction_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    """mean / sum / amax over `dim`: the reduced dimensions stay whole, every other one may be split."""
    ops = tensor_operands(node)
    shape_out = node_shape(node)
    if len(ops) != 1 or shape_out is None:
        return [_replicated_strategy(node, ctx)]
    x = ops[0]
    xs = node_shape(x)
    dim = node.kwargs.get("dim", node.args[1] if len(node.args) > 1 else None)
    keep = node.kwargs.get("keepdim", node.args[2] if len(node.args) > 2 else False)
    if dim is None:
        return [_replicated_strategy(node, ctx)]
    dims = {d % len(xs) for d in ([dim] if isinstance(dim, int) else dim)}
    out = []
    for spec in enumerate_specs(xs, ctx.mesh_shape, allowed_dims=[d for d in range(len(xs)) if d not in dims]):
        ospec = tuple(a for d, a in enumerate(spec) if keep or d not in dims)
        if keep:
            ospec = tuple(None if d in dims else a for d, a in enumerate(spec))
        f = shard_factor(spec, ctx.mesh_shape)
        out.append(ShardingStrategy(f"reduce{spec_str(spec)}", ospec, {x.name: spec},
                                    compute_cost=ctx.mem_time(node_bytes(x), f), memory_cost=node_bytes(node) / f))
    return out


def reshape_dim_map(in_shape: Sequence[int], out_shape: Sequence[int]) -> Optional[Dict[int, Tuple[int, bool]]]:
    """For every input dimension: (output dimension that starts the same contiguous group, is-leading-in-its-group).
    Groups are the maximal runs of input / output dimensions with equal element counts."""
    if math.prod(in_shape) != math.prod(out_shape) or 0 in in_shape:
        return None
    i = j = 0
    mapping: Dict[int, Tuple[int, bool]] = {}
    ni, nj = len(in_shape), len(out_shape)
    while i < ni and j < nj:
        gi, gj = [i], [j]
        pi, pj = in_shape[i], out_shape[j]
        i, j = i + 1, j + 1
        while pi != pj:
            if pi < pj:
                if i >= ni:
                    return None
                pi *= in_shape[i]
                gi.append(i)
                i += 1
            else:
                if j >= nj:
                    return None
                pj *= out_shape[j]
                gj.append(j)
                j += 1
        # size-1 dimensions at the head of a group cannot carry a shard: lead = first dimension with extent > 1
        lead_in = next((d for d in gi if in_shape[d] > 1), gi[0])
        lead_out = next((d for d in gj if out_shape[d] > 1), gj[0])
        for d in gi:
            mapping[d] = (lead_out, d == lead_in)
    while i < ni:                                 # trailing size-1 input dimensions
        mapping[i] = (nj - 1, False)
        i += 1
    return mapping


RESHAPE_METHODS = {"view", "reshape", "flatten", "unsqueeze", "squeeze", "unflatten"}


def reshape_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    ops = tensor_operands(node)
    out_shape = node_shape(node)
    if len(ops) != 1 or out_shape is None:
        return [_replicated_strategy(node, ctx)]
    x = ops[0]
    xs = node_shape(x)
    mapping = reshape_dim_map(xs, out_shape)
    out = []
    for spec in enumerate_specs(xs, ctx.mesh_shape):
        ospec: List[Optional[int]] = [None] * len(out_shape)
        ok = True
        for d, a in enumerate(spec):
            if a is None:
                continue
            if mapping is None or d not in mapping or not mapping[d][1]:
                ok = False
                break
            od = mapping[d][0]
            if out_shape[od] % ctx.mesh_shape[a] or ospec[od] is not None:
                ok = False
                break
            ospec[od] = a
        if ok:
            out.append(ShardingStrategy(f"reshape{spec_str(spec)}", tuple(ospec), {x.name: spec},
                                        memory_cost=0.0))
    return out or [_replicated_strategy(node, ctx)]


def permute_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    ops = tensor_operands(node)
    out_shape = node_shape(node)
    if len(ops) != 1 or out_shape is None:
        return [_replicated_strategy(node, ctx)]
    x = ops[0]
    nd = len(node_shape(x))
    name = node.target if isinstance(node.target, str) else getattr(node.target, "__name__", "")
    if name in ("transpose", "swapaxes"):
        d0, d1 = node.args[1] % nd, node.args[2] % nd
        perm = list(range(nd))
        perm[d0], perm[d1] = perm[d1], perm[d0]
    elif name == "t":
        perm = list(range(nd))[::-1]
    else:
        dims = node.args[1:] if not isinstance(node.args[1], (tuple, list)) else node.args[1]
        if node.kwargs.get("dims") is not None:
            dims = node.kwargs["dims"]
        perm = [d % nd for d in dims]
    out = []
    for spec in enumerate_specs(node_shape(x), ctx.mesh_shape):
        out.append(ShardingStrategy(f"permute{spec_str(spec)}", tuple(spec[p] for p in perm), {x.name: spec}))
    return out


def size_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    """`x.size()` / `x.shape`: free under every layout of `x` — the runtime pass reports GLOBAL extents (local extent
    times the mesh axis size) so shape arithmetic in the graph keeps its single-device meaning."""
    ops = tensor_operands(node)
    if len(ops) != 1:
        return [_replicated_strategy(node, ctx)]
    x = ops[0]
    return [ShardingStrategy(f"size{spec_str(s)}", None, {x.name: s}) for s in enumerate_specs(node_shape(x), ctx.mesh_shape)]


def _role_products(axes: Sequence[int], roles: Sequence) -> List[Dict[int, object]]:
    out = []
    for assign in itertools.product(roles, repeat=len(axes)):
        used = [r for r in assign if r is not None]
        if len(set(used)) != len(used):
            continue
        out.append({a: r for a, r in zip(axes, assign)})
    return out


def linear_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    """y[..., N] = x[..., K] W[N, K]^T + b.  Roles of a mesh axis: split a batch dimension of x (data parallel), split
    N (column parallel: x must be whole, dgrad is a partial sum), split K (row parallel: the result is a partial sum)."""
    mod = ctx.gm.get_submodule(node.target)
    ops = tensor_operands(node)
    if len(ops) != 1 or node_shape(node) is None:
        return [_replicated_strategy(node, ctx)]
    x = ops[0]
    xs, ys = node_shape(x), node_shape(node)
    nd = len(xs)
    K, N = mod.in_features, mod.out_features
    M = math.prod(xs[:-1])
    flops = 2.0 * M * K * N
    wbytes = float(K * N) * mod.weight.element_size()
    xbytes, ybytes = node_bytes(x), node_bytes(node)
    ms = ctx.mesh_shape
    out = []
    for roles in _role_products(_axes(ms), [None, "col", "row"] + list(range(nd - 1))):
        in_spec: List[Optional[int]] = [None] * nd
        out_spec: List[Optional[int]] = [None] * nd
        col = row = None
        batch_axes = []
        ok = True
        for a, r in roles.items():
            if r is None:
                continue
            if r == "col":
                ok &= N % ms[a] == 0
                col = a
                out_spec[-1] = a
            elif r == "row":
                ok &= K % ms[a] == 0
                row = a
                in_spec[-1] = a
            else:
                ok &= xs[r] % ms[a] == 0 and xs[r] >= ms[a]
                in_spec[r] = out_spec[r] = a
                batch_axes.append(a)
        if not ok:
            continue
        bf = math.prod(ms[a] for a in batch_axes) if batch_axes else 1
        cf = ms[col] if col is not None else 1
        rf = ms[row] if row is not None else 1
        comm = 0.0
        if row is not None:
            comm += ctx.mesh.all_reduce_cost(ybytes / (bf * cf), row)
        if col is not None and ctx.train:
            comm += ctx.mesh.all_reduce_cost(xbytes / (bf * rf), col)
        if ctx.train:
            comm += sum(ctx.mesh.all_reduce_cost(wbytes / (cf * rf), a) for a in batch_axes)
        params = {"weight": (col, row)}
        if mod.bias is not None:
            params["bias"] = (col,)
        tag = "+".join(f"{r if isinstance(r, str) else 'b' + str(r)}@{a}" for a, r in roles.items() if r is not None)
        out.append(ShardingStrategy(
            tag or "replicate", tuple(out_spec), {x.name: tuple(in_spec)}, params,
            compute_cost=ctx.mm_time(flops, bf * cf * rf), comm_cost=comm,
            memory_cost=wbytes / (cf * rf) + ybytes / (bf * cf),
            reduce_axes=() if row is None else (row,),
            bwd_reduce_inputs={x.name: (col,)} if (col is not None and ctx.train) else {},
            grad_sync_axes=tuple(batch_axes)))
    return out


def embedding_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    mod = ctx.gm.get_submodule(node.target)
    ops = tensor_operands(node)
    if len(ops) != 1 or node_shape(node) is None:
        return [_replicated_strategy(node, ctx)]
    ids = ops[0]
    ishape = node_shape(ids)
    nd = len(ishape)
    H = mod.embedding_dim
    wbytes = float(mod.num_embeddings * H) * mod.weight.element_size()
    ybytes = node_bytes(node)
    ms = ctx.mesh_shape
    out = []
    for roles in _role_products(_axes(ms), [None, "hidden"] + list(range(nd))):
        in_spec: List[Optional[int]] = [None] * nd
        out_spec: List[Optional[int]] = [None] * (nd + 1)
        hid, batch_axes, ok = None, [], True
        for a, r in roles.items():
            if r is None:
                continue
            if r == "hidden":
                ok &= H % ms[a] == 0
                hid = a
                out_spec[-1] = a
            else:
                ok &= ishape[r] % ms[a] == 0 and ishape[r] >= ms[a]
                in_spec[r] = out_spec[r] = a
                batch_axes.append(a)
        if not ok:
            continue
        bf = math.prod(ms[a] for a in batch_axes) if batch_axes else 1
        hf = ms[hid] if hid is not None else 1
        comm = sum(ctx.mesh.all_reduce_cost(wbytes / hf, a) for a in batch_axes) if ctx.train else 0.0
        tag = "+".join(f"{r if isinstance(r, str) else 'b' + str(r)}@{a}" for a, r in roles.items() if r is not None)
        out.append(ShardingStrategy(tag or "replicate", tuple(out_spec), {ids.name: tuple(in_spec)},
                                    {"weight": (None, hid)}, compute_cost=ctx.mem_time(2 * ybytes, bf * hf),
                                    comm_cost=comm, memory_cost=wbytes / hf + ybytes / (bf * hf),
                                    grad_sync_axes=tuple(batch_axes)))
    return out


def layernorm_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    mod = ctx.gm.get_submodule(node.target)
    ops = tensor_operands(node)
    shape = node_shape(node)
    if len(ops) != 1 or shape is None:
        return [_replicated_strategy(node, ctx)]
    x = ops[0]
    k = len(mod.normalized_shape)
    nbytes = node_bytes(node)
    pbytes = sum(p.numel() * p.element_size() for p in mod.parameters())
    out = []
    for spec in enumerate_specs(shape, ctx.mesh_shape, allowed_dims=list(range(len(shape) - k))):
        f = shard_factor(spec, ctx.mesh_shape)
        axes = _used_axes(spec)
        comm = sum(ctx.mesh.all_reduce_cost(pbytes, a) for a in axes) if (ctx.train and pbytes) else 0.0
        params = {n: replicated(p.dim()) for n, p in mod.named_parameters(recurse=False)}
        out.append(ShardingStrategy(f"norm{spec_str(spec)}", spec, {x.name: spec}, params,
                                    compute_cost=ctx.mem_time(2 * nbytes, f), comm_cost=comm,
                                    memory_cost=pbytes + nbytes / f, grad_sync_axes=axes))
    return out


def matmul_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    """A[..., M, K] @ B[..., K, N] with identical leading dimensions (attention scores / context)."""
    ops = tensor_operands(node)
    ys = node_shape(node)
    if len(ops) != 2 or ys is None or ops[0] is ops[1]:
        return [_replicated_strategy(node, ctx)]
    A, B = ops
    sa, sb = node_shape(A), node_shape(B)
    if len(sa) != len(sb) or len(sa) < 2 or sa[:-2] != sb[:-2]:
        return [_replicated_strategy(node, ctx)]
    nd = len(sa)
    M, K, N = sa[-2], sa[-1], sb[-1]
    lead = math.prod(sa[:-2])
    flops = 2.0 * lead * M * K * N
    ms = ctx.mesh_shape
    out = []
    for roles in _role_products(_axes(ms), [None, "m", "n", "k"] + list(range(nd - 2))):
        a_spec: List[Optional[int]] = [None] * nd
        b_spec: List[Optional[int]] = [None] * nd
        y_spec: List[Optional[int]] = [None] * nd
        red, bwd_a, bwd_b, ok, f = [], [], [], True, 1
        for ax, r in roles.items():
            if r is None:
                continue
            f *= ms[ax]
            if r == "m":
                ok &= M % ms[ax] == 0
                a_spec[-2] = y_spec[-2] = ax
                bwd_b.append(ax)
            elif r == "n":
                ok &= N % ms[ax] == 0
                b_spec[-1] = y_spec[-1] = ax
                bwd_a.append(ax)
            elif r == "k":
                ok &= K % ms[ax] == 0
                a_spec[-1] = b_spec[-2] = ax
                red.append(ax)
            else:
                ok &= sa[r] % ms[ax] == 0 and sa[r] >= ms[ax]
                a_spec[r] = b_spec[r] = y_spec[r] = ax
        if not ok:
            continue
        ybytes = node_bytes(node)
        comm = sum(ctx.mesh.all_reduce_cost(ybytes * ms[ax] / f, ax) for ax in red)
        bwd = {}
        if ctx.train:
            if bwd_a:
                bwd[A.name] = tuple(bwd_a)
                comm += sum(ctx.mesh.all_reduce_cost(node_bytes(A), ax) for ax in bwd_a)
            if bwd_b:
                bwd[B.name] = tuple(bwd_b)
                comm += sum(ctx.mesh.all_reduce_cost(node_bytes(B), ax) for ax in bwd_b)
        tag = "+".join(f"{r if isinstance(r, str) else 'b' + str(r)}@{ax}" for ax, r in roles.items() if r is not None)
        out.append(ShardingStrategy(tag or "replicate", tuple(y_spec), {A.name: tuple(a_spec), B.name: tuple(b_spec)},
                                    compute_cost=ctx.mm_time(flops, f), comm_cost=comm,
                                    memory_cost=ybytes / shard_factor(tuple(y_spec), ms), reduce_axes=tuple(red),
                                    bwd_reduce_inputs=bwd))
    return out


def fallback_handler(node: fx.Node, ctx: HandlerContext) -> List[ShardingStrategy]:
    return [_replicated_strategy(node, ctx, cost=ctx.mem_time(2 * node_bytes(node), 1))]


# ---------------------------------------------------------------------------------------------------------- registry
_MODULE_HANDLERS: Dict[type, Callable] = {}
_FUNCTION_HANDLERS: Dict[object, Callable] = {}
_METHOD_HANDLERS: Dict[str, Callable] = {}


def register_module_handler(*types: type):
    def deco(fn):
        for t in types:
            _MODULE_HANDLERS[t] = fn
        return fn
    return deco


def register_function_handler(*targets):
    def deco(fn):
        for t in targets:
            (_METHOD_HANDLERS if isinstance(t, str) else _FUNCTION_HANDLERS)[t] = fn
        return fn
    return deco


register_module_handler(nn.Linear)(linear_handler)
register_module_handler(nn.Embedding)(embedding_handler)
register_module_handler(nn.LayerNorm)(layernorm_handler)
register_module_handler(nn.Softmax, nn.LogSoftmax)(softmax_handler)
register_module_handler(nn.ReLU, nn.GELU, nn.SiLU, nn.Tanh, nn.Sigmoid, nn.Dropout, nn.Identity, nn.LeakyReLU,
                        nn.ELU, nn.Softplus, nn.Mish, nn.Hardtanh, nn.ReLU6)(elementwise_handler)

_POINTWISE_FUNCS = [operator.add, operator.sub, operator.mul, operator.truediv, operator.neg, operator.pow, torch.add,
                    torch.sub, torch.mul, torch.div, torch.neg, torch.pow, torch.rsqrt, torch.sqrt, torch.exp,
                    torch.tanh, torch.sigmoid, torch.relu, torch.abs, torch.square, F.relu, F.gelu, F.silu, F.dropout,
                    F.tanh, F.sigmoid, F.leaky_relu, F.elu, F.softplus, F.mish, torch.clone, torch.where,
                    torch.maximum, torch.minimum, torch.clamp]
register_function_handler(*_POINTWISE_FUNCS)(elementwise_handler)
register_function_handler("add", "sub", "mul", "div", "neg", "pow", "rsqrt", "sqrt", "exp", "tanh", "sigmoid", "relu",
                          "abs", "square", "contiguous", "clone", "to", "float", "half", "bfloat16", "type_as",
                          "clamp", "masked_fill", "detach", "add_", "mul_")(elementwise_handler)
register_function_handler(F.softmax, F.log_softmax, torch.softmax, torch.log_softmax, "softmax", "log_softmax")(
    softmax_handler)
register_function_handler(torch.mean, torch.sum, torch.amax, "mean", "sum", "amax")(reduction_handler)
register_function_handler(torch.reshape, torch.flatten, torch.unsqueeze, torch.squeeze, *RESHAPE_METHODS)(
    reshape_handler)
register_function_handler(torch.transpose, torch.permute, torch.swapaxes, "transpose", "permute", "swapaxes", "t")(
    permute_handler)
register_function_handler(torch.matmul, torch.bmm, operator.matmul, "matmul", "bmm")(matmul_handler)
register_function_handler("size")(size_handler)


def generate_strategies(node: fx.Node, ctx: HandlerContext) -> StrategiesVector:
    if node.op == "placeholder":
        strategies = placeholder_handler(node, ctx)
    elif node.op == "get_attr":
        strategies = get_attr_handler(node, ctx)
    elif node.op == "output":
        strategies = output_handler(node, ctx)
    elif node.op == "call_module":
        mod = ctx.gm.get_submodule(node.target)
        fn = next((h for t, h in _MODULE_HANDLERS.items() if type(mod) is t), None) or \
            next((h for t, h in _MODULE_HANDLERS.items() if isinstance(mod, t)), fallback_handler)
        strategies = fn(node, ctx)
    elif node.op == "call_function":
        if node.target is getattr and len(node.args) == 2 and node.args[1] == "shape":
            strategies = size_handler(node, ctx)
        else:
            strategies = _FUNCTION_HANDLERS.get(node.target, fallback_handler)(node, ctx)
    elif node.op == "call_method":
        strategies = _METHOD_HANDLERS.get(node.target, fallback_handler)(node, ctx)
    else:
        strategies = fallback_handler(node, ctx)
    vec = StrategiesVector(node)
    vec.extend(strategies)
    return vec
