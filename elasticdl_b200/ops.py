"""Device primitives of the client side of the exchange, as torch-level calls
into libb200ps.so: first-occurrence unique (tf.unique), row gather and its
backward (segment sum with warp-level id dedup), and the pooled lookup of sparse
input (prep, combine and its backward).  CUDA only -- no fallback."""
import ctypes

import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import check

_ws = {}


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _need_cuda(t, what):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError("%s must be a CUDA tensor: elasticdl_b200 has no CPU path" % what)


def unique(ids, T=1):
    """tf.unique (elasticdl/python/elasticdl/embedding_delegate.py:85) over T
    equal-length segments.  ids: int64 CUDA tensor of T*k elements.
    Returns (uniq int64 [T*k] (first n_unique[t] of each segment valid, first-
    occurrence order), inv int32 [T*k], n_unique int32 [T]) -- nothing is read
    back to the host."""
    _need_cuda(ids, "ids")
    ids = ids.contiguous().view(-1)
    if ids.dtype != torch.int64:
        ids = ids.to(torch.int64)
    k = ids.numel() // T
    lib = _lib.lib()
    need = lib.b200ps_unique_workspace(T, k)
    # one workspace per (device, stream): two worker threads on different streams must never share
    # the position / key arrays (a stale one is dropped once its stream has run past the last use)
    stream = torch.cuda.current_stream(ids.device)
    key = (ids.device, stream.cuda_stream)
    ws = _ws.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(need, dtype=torch.uint8, device=ids.device)
        if key in _ws:
            _ws[key].record_stream(stream)
        _ws[key] = ws
    uniq = torch.empty(T * k, dtype=torch.int64, device=ids.device)
    inv = torch.empty(T * k, dtype=torch.int32, device=ids.device)
    n_unique = torch.empty(T, dtype=torch.int32, device=ids.device)
    with torch.cuda.device(ids.device):
        check(lib.b200ps_unique(None, ids.data_ptr(), T, k, uniq.data_ptr(), inv.data_ptr(), n_unique.data_ptr(),
                                ws.data_ptr(), ws.numel(), _stream(ids.device)))
    return uniq, inv, n_unique


def gather_rows(bet, inv, T, k, dim):
    """out[t, i, :] = bet[t, inv[t, i], :]   (tf.gather(batch_embedding, idx), embedding_delegate.py:95).
    bet is [T, R, dim] with R == k rows allocated per segment."""
    _need_cuda(bet, "bet")
    out = torch.empty((T * k, dim), dtype=torch.float32, device=bet.device)
    with torch.cuda.device(bet.device):
        check(_lib.lib().b200ps_gather_rows(None, bet.data_ptr(), inv.data_ptr(), T, k, dim, out.data_ptr(),
                                            _stream(bet.device)))
    return out


def segment_sum(values, inv, T, k, dim):
    """out[t, inv[t, i], :] += values[t, i, :]: the sum deduplicate_indexed_slices
    computes (python/common/tensor_utils.py:39-60) == the gradient of gather_rows."""
    _need_cuda(values, "values")
    values = values.contiguous()
    out = torch.empty((T * k, dim), dtype=torch.float32, device=values.device)
    with torch.cuda.device(values.device):
        check(_lib.lib().b200ps_segment_sum(None, values.data_ptr(), inv.data_ptr(), T, k, dim, out.data_ptr(),
                                            _stream(values.device)))
    return out


COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}


def sparse_prep(rows, vals, batch, dim):
    """_prune_invalid_ids + sparse_fill_empty_rows(ids, 0) (embedding_delegate.py:155-170) of a coalesced
    [batch, L] COO (rows int64 [nnz] row-major, vals int64 | int32 [nnz]), in three launches with no host read.
    Returns (ids int64 [nnz + batch]: the filled id stream, then copies of its last id; ws: the workspace the
    combine reads, whose first int32 counts the entries dropped for a row outside [0, batch))."""
    _need_cuda(vals, "vals")
    nnz = vals.numel()
    rows = rows.contiguous().view(-1)
    vals = vals.contiguous().view(-1)
    if vals.dtype not in (torch.int32, torch.int64):
        vals = vals.to(torch.int64)
    lib = _lib.lib()
    need = lib.b200ps_sparse_workspace(batch, nnz, dim)
    ws = torch.empty(need, dtype=torch.uint8, device=vals.device)
    ids = torch.empty(nnz + batch, dtype=torch.int64, device=vals.device)
    with torch.cuda.device(vals.device):
        check(lib.b200ps_sparse_prep(None, rows.data_ptr() if nnz else None, vals.data_ptr() if nnz else None,
                                     int(vals.dtype == torch.int32), batch, nnz, dim, ids.data_ptr(), ws.data_ptr(),
                                     need, _stream(vals.device)))
    return ids, ws


def bag_prep(group, input, offsets, dim, include_last_offset=False, padding_idx=None):
    """nn.EmbeddingBag's two input forms -> the (ids, ws) sparse_prep gives for the equivalent [B, L] COO, in one launch
    with no host read: `input` int64 | int32 [B, L] with offsets None, or 1-D ids with int64 | int32 `offsets` [B]
    ([B + 1] with include_last_offset).  Entries equal to padding_idx are dropped; bad offsets and negative ids set the
    error word of `group` (a PSGroup), so group.check() raises.  Returns (ids, ws, B, nnz) for SparseCombine."""
    _need_cuda(input, "input")
    if input.dtype not in (torch.int32, torch.int64):
        raise ValueError("EmbeddingBag input must be int32 or int64, not %s" % input.dtype)
    if offsets is None:
        if input.dim() != 2:
            raise ValueError("EmbeddingBag input without offsets must be 2-D [B, L], not %s" % (tuple(input.shape),))
        batch, width = int(input.shape[0]), int(input.shape[1])
        offs = None
    else:
        if input.dim() != 1 or offsets.dim() != 1:
            raise ValueError("EmbeddingBag input with offsets must be 1-D ids and 1-D offsets")
        _need_cuda(offsets, "offsets")
        offs = offsets.contiguous() if offsets.dtype == torch.int64 else offsets.to(torch.int64)
        batch, width = int(offs.numel()) - (1 if include_last_offset else 0), -1
    if batch < 1:
        raise ValueError("EmbeddingBag input has no bag")
    vals = input.contiguous().view(-1)
    nnz = vals.numel()
    lib = _lib.lib()
    need = lib.b200ps_sparse_workspace(batch, nnz, dim)
    ws = torch.empty(need, dtype=torch.uint8, device=vals.device)
    ids = torch.empty(nnz + batch, dtype=torch.int64, device=vals.device)
    with torch.cuda.device(vals.device):
        check(lib.b200ps_bag_prep(group._h, vals.data_ptr() if nnz else None, int(vals.dtype == torch.int32),
                                  offs.data_ptr() if offs is not None else None, width, int(bool(include_last_offset)),
                                  -1 if padding_idx is None else int(padding_idx), batch, nnz, dim, ids.data_ptr(),
                                  ws.data_ptr(), need, _stream(vals.device)))
    return ids, ws, batch, nnz


class SparseCombine(torch.autograd.Function):
    """BET [U, dim] -> [batch, dim]: each row's BET rows summed, scaled by the combiner, 0 for the rows that were
    empty (sparse_segment_{sum,mean,sqrt_n}); backward = the scaled segment sum into [U, dim].  dim is the one
    sparse_prep sized `ws` for.

    weights (optional): float32 [nnz] in input-entry order (the coalesced COO's values, or the bag input's): row b is
    sum w_j e_j, divided by sum w_j (mean) or sqrt(sum w_j^2) (sqrtn).  Weights that require grad get the gradient of
    the sum combiner (0 for the entries prep dropped); under mean and sqrtn they are data, as in the reference's
    weighted feature columns, and weights that require grad raise ValueError."""

    @staticmethod
    def forward(ctx, bet, inv, ws, batch, nnz, combiner, dim, weights=None):
        bet = bet.contiguous()
        if bet.dim() != 2 or bet.shape[1] != dim:
            raise ValueError("the lookup returned rows of shape %s, the layer needs [n_unique, %d]"
                             % (tuple(bet.shape), dim))
        comb = COMBINERS[combiner]
        lib = _lib.lib()
        out = torch.empty((batch, dim), dtype=torch.float32, device=bet.device)
        if weights is None:
            ctx.save_for_backward(inv, ws)
        else:
            if ctx.needs_input_grad[7] and combiner != "sum":
                raise ValueError("weights that require grad need the sum combiner (under %s they are data)" % combiner)
            _need_cuda(weights, "weights")
            if weights.numel() != nnz:
                raise ValueError("%d weights for %d input entries" % (weights.numel(), nnz))
            weights = weights.detach().reshape(-1).to(torch.float32).contiguous()
            ctx.save_for_backward(inv, ws, weights, bet if ctx.needs_input_grad[7] else None)
        ctx.shape = (batch, nnz, dim, comb, bet.shape[0])
        with torch.cuda.device(bet.device):
            if weights is None:
                check(lib.b200ps_sparse_combine(None, bet.data_ptr(), inv.data_ptr(), ws.data_ptr(), ws.numel(), batch,
                                                nnz, dim, comb, out.data_ptr(), _stream(bet.device)))
            else:
                check(lib.b200ps_sparse_combine_weighted(None, bet.data_ptr(), inv.data_ptr(), weights.data_ptr(),
                                                         ws.data_ptr(), ws.numel(), batch, nnz, dim, comb,
                                                         out.data_ptr(), _stream(bet.device)))
        return out

    @staticmethod
    def backward(ctx, grad_out):
        inv, ws, *wsaved = ctx.saved_tensors
        batch, nnz, dim, comb, u = ctx.shape
        g = grad_out.contiguous()
        gbet = torch.empty((u, dim), dtype=torch.float32, device=g.device)
        lib = _lib.lib()
        with torch.cuda.device(g.device):
            if not wsaved:
                check(lib.b200ps_sparse_combine_grad(None, g.data_ptr(), inv.data_ptr(), ws.data_ptr(), ws.numel(),
                                                     batch, nnz, dim, comb, u, gbet.data_ptr(), _stream(g.device)))
                return gbet, None, None, None, None, None, None, None
            weights, bet = wsaved
            gw = torch.empty(nnz, dtype=torch.float32, device=g.device) if bet is not None else None
            check(lib.b200ps_sparse_combine_weighted_grad(
                None, g.data_ptr(), inv.data_ptr(), weights.data_ptr(), bet.data_ptr() if bet is not None else None,
                ws.data_ptr(), ws.numel(), batch, nnz, dim, comb, u, gbet.data_ptr(),
                gw.data_ptr() if gw is not None else None, _stream(g.device)))
        return gbet, None, None, None, None, None, None, gw


class GatherRows(torch.autograd.Function):
    """BET[U(+pad), dim] -> rows per id occurrence; backward = segment_sum."""

    @staticmethod
    def forward(ctx, bet, inv, T, k, dim):
        ctx.save_for_backward(inv)
        ctx.shape = (T, k, dim, bet.shape)
        bet_c = bet.contiguous()
        if bet_c.numel() != T * k * dim:
            # exact-shape BET ([U, dim], T == 1): pad to k rows so segments stay addressable
            pad = torch.zeros((T * k, dim), dtype=torch.float32, device=bet.device)
            pad[: bet_c.shape[0]] = bet_c
            bet_c = pad
        return gather_rows(bet_c, inv, T, k, dim)

    @staticmethod
    def backward(ctx, grad_out):
        (inv,) = ctx.saved_tensors
        T, k, dim, shape = ctx.shape
        g = segment_sum(grad_out.reshape(T * k, dim), inv, T, k, dim)
        if g.numel() != int(torch.Size(shape).numel()):
            g = g[: shape[0]]
        return g.reshape(shape), None, None, None, None
