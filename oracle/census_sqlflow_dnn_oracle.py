"""Float64 reference of a feature-column DNN step by table kind -- TEST INFRASTRUCTURE.

census_model_sqlflow/dnn (model_zoo/census_model_sqlflow/dnn/census_functional.py:28-70) is census_dnn_model's
DenseFeatures -> Dense(16, relu) x2 -> Dense(1, sigmoid) with the per-sample binary cross-entropy (batch sums, Q16),
so its tower is oracle/fc_dnn_oracle.py's, unchanged.  What the table kind (fc_dnn.Layout.table_kinds, carried by
spec()["table_kinds"]) changes is where the rows live and how they move (DESIGN.md section 4, Q36):
  * ids: Fingerprint64 % rows of the raw string (oracle/feature_oracle.py), "" to the fill id 0 (Q18);
  * a "dense" table is one [rows, dim] dense PS parameter whose pushed IndexedSlices -- the batch's unique ids and
    their summed rows, the fill id 0 with a zero row included -- are applied by the PS's Indexed Adam
    (go/pkg/ps/optimizer.go Indexed kernels, kernel_api.cc:40-77): m, v and the row of each pushed id move, every
    other row and its slots stay as they were;
  * a "ps" table (census_dnn_model) is a hashed PS table whose Sparse Adam applies the same per-row formula to the
    same rows.
Plain torch float64, device-agnostic.
"""
import math

import numpy as np
import torch

from oracle import feature_oracle as FO


def ids_from_strings(raw, rows):
    """A hash-bucket column's ids from raw strings (a list of bytes or str): Fingerprint64 % rows, and "" to the
    fill id 0 that safe_embedding_lookup_sparse looks an empty sample up with (Q18).  int64 numpy [B]."""
    raw = [s.encode() if isinstance(s, str) else bytes(s) for s in raw]
    return np.where([len(s) == 0 for s in raw], 0, FO.hashing(raw, rows)).astype(np.int64)


def indexed_adam(p, m, v, ids, g, lr, step, beta1=0.9, beta2=0.999, epsilon=1e-7):
    """The PS's Indexed Adam of one dense parameter [rows, dim] in float64: for each unique id in `ids` with its
    summed gradient row g[i], m = b1 m + (1 - b1) g, v = b2 v + (1 - b2) g^2, p -= lr_t m / (sqrt(v) + eps) with
    lr_t = lr sqrt(1 - b2^step) / (1 - b1^step) (step: the shard's step after the push's bump, Q2).  Returns new
    float64 (p, m, v); the rows not in `ids` are exact float64 copies of the inputs'."""
    p, m, v = (torch.as_tensor(t).to(torch.float64).clone() for t in (p, m, v))
    ids = torch.as_tensor(ids).long().to(p.device)
    if ids.numel() != torch.unique(ids).numel():
        raise ValueError("an Indexed update takes unique ids (PSClient deduplicates the IndexedSlices first)")
    g = torch.as_tensor(g).to(device=p.device, dtype=torch.float64).reshape(ids.numel(), p.shape[1])
    b1, b2, eps = (float(np.float32(x)) for x in (beta1, beta2, epsilon))  # the PS parses them as float32
    lr_t = float(lr) * math.sqrt(1.0 - b2 ** step) / (1.0 - b1 ** step)
    m[ids] = b1 * m[ids] + (1 - b1) * g
    v[ids] = b2 * v[ids] + (1 - b2) * g * g
    p[ids] = p[ids] - lr_t * m[ids] / (v[ids].sqrt() + eps)
    return p, m, v


def apply_dense_tables(spec, state, uniq, gsum, lr, step, **adam):
    """Indexed Adam on every "dense" table of `spec`.  state: {k: (p, m, v)} of table k; uniq[k]: its unique ids,
    gsum[k]: their summed gradient rows (the tower's, in the same order).  Returns the new {k: (p, m, v)}."""
    out = {}
    for k, kind in enumerate(spec["table_kinds"]):
        if kind == "dense":
            out[k] = indexed_adam(*state[k], uniq[k], gsum[k], lr, step, **adam)
    return out
