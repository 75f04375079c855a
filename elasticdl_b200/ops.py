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


class SparseCombine(torch.autograd.Function):
    """BET [U, dim] -> [batch, dim]: each row's BET rows summed, scaled by the combiner, 0 for the rows that were
    empty (sparse_segment_{sum,mean,sqrt_n}); backward = the scaled segment sum into [U, dim].  dim is the one
    sparse_prep sized `ws` for."""

    @staticmethod
    def forward(ctx, bet, inv, ws, batch, nnz, combiner, dim):
        bet = bet.contiguous()
        if bet.dim() != 2 or bet.shape[1] != dim:
            raise ValueError("the lookup returned rows of shape %s, the layer needs [n_unique, %d]"
                             % (tuple(bet.shape), dim))
        ctx.save_for_backward(inv, ws)
        ctx.shape = (batch, nnz, dim, COMBINERS[combiner], bet.shape[0])
        out = torch.empty((batch, dim), dtype=torch.float32, device=bet.device)
        with torch.cuda.device(bet.device):
            check(_lib.lib().b200ps_sparse_combine(None, bet.data_ptr(), inv.data_ptr(), ws.data_ptr(), ws.numel(), batch,
                                                   nnz, dim, COMBINERS[combiner], out.data_ptr(), _stream(bet.device)))
        return out

    @staticmethod
    def backward(ctx, grad_out):
        inv, ws = ctx.saved_tensors
        batch, nnz, dim, comb, u = ctx.shape
        g = grad_out.contiguous()
        gbet = torch.empty((u, dim), dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            check(_lib.lib().b200ps_sparse_combine_grad(None, g.data_ptr(), inv.data_ptr(), ws.data_ptr(), ws.numel(),
                                                        batch, nnz, dim, comb, u, gbet.data_ptr(), _stream(g.device)))
        return gbet, None, None, None, None, None, None


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
