"""ElasticDL Embedding layer over the HBM parameter server (torch module).

Public surface of elasticdl/python/elasticdl/layers/embedding.py:20-162 and the
EmbeddingDelegate it wraps (embedding_delegate.py:26-310): same constructor
arguments, `set_lookup_embedding_func`, `set_tape`, `reset`, `embedding_and_ids`,
`embedding_weight_name`, `set_embedding_weight_name`; dense and sparse (combiner
sum / mean / sqrtn) inputs.

Differences that follow from torch (documented in DESIGN.md):
  * there is no GradientTape: `set_tape(x)` with a truthy x makes the layer
    record the batch embedding tensor (BET) with requires_grad, which is what
    watching it on the tape does (embedding_delegate.py:266-281);
  * torch has no IndexedSlices: BET.grad is the dense [U, dim] gradient, i.e. the
    per-occurrence rows already summed per unique id -- the sum PSClient computes
    next anyway (ps_client.py:255-257) -- so `batch_ids` holds the UNIQUE ids that
    index BET rows (the reference stores the flat ids and pairs them with the
    IndexedSlices values).
"""
import collections

import torch

from elasticdl_b200 import ops

EmbeddingAndIds = collections.namedtuple("EmbeddingAndIds", ["batch_embedding", "batch_ids"])

_layer_counter = collections.Counter()


class Embedding(torch.nn.Module):
    """
    Input: indexes for the embedding entries with a shape of (batch_size, input_length);
      a dense int tensor, or a sparse COO tensor [batch, max_len] (combiner required).
    Output: (batch_size, input_length, output_dim) if combiner is None,
            (batch_size, output_dim) for sparse input with a combiner.
    """

    def __init__(self, output_dim, input_dim=None, embeddings_initializer="uniform", mask_zero=False,
                 input_length=None, combiner=None, name=None, **kwargs):
        super().__init__()
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.embeddings_initializer = embeddings_initializer
        self.mask_zero = mask_zero
        self.supports_masking = mask_zero
        self.input_length = input_length
        self.combiner = combiner
        if name is None:  # keras-style auto naming: embedding, embedding_1, ...
            n = _layer_counter["embedding"]
            _layer_counter["embedding"] += 1
            name = "embedding" if n == 0 else "embedding_%d" % n
        self._name = name
        self.embedding_weight_name = self._name + "/embeddings:0"
        self._lookup_embedding_func = None
        self._embedding_and_ids = []
        self.tape = None
        # batched lookups (worker/ps_trainer.py): which input object this layer was called with in the
        # current step, and -- when the trainer looked all layers up in one launch before the forward
        # pass -- (that input object, this layer's rows of the batched result)
        self._inputs_seen = []
        self._prefetched = None

    @property
    def name(self):
        return self._name

    @staticmethod
    def get_key(name_list):
        return "-".join(map(str, name_list))

    # -------------------------------------------------------------- delegate API
    def set_lookup_embedding_func(self, func):
        """func(layer_name, embedding_id_list) -> [len(ids), output_dim] (layers/embedding.py:146-155)."""
        self._lookup_embedding_func = func

    def set_tape(self, tape):
        self.tape = tape

    def reset(self):
        self.tape = None
        self._embedding_and_ids = []
        self._inputs_seen = []
        self._prefetched = None

    @property
    def embedding_and_ids(self):
        return self._embedding_and_ids

    def set_embedding_weight_name(self, name):
        self.embedding_weight_name = name

    def compute_mask(self, inputs, mask=None):
        if inputs.is_sparse:
            raise ValueError("SparseTensor inputs do not support mask_zero")
        if not self.supports_masking:
            return None
        return inputs != 0

    # -------------------------------------------------------------- lookup
    def _check_id_valid(self, unique_ids):
        """embedding_delegate.py:254-264 (raises only when an id exceeds input_dim)."""
        if not self.input_dim:
            return
        mx = int(unique_ids.max().item())
        if mx > self.input_dim:
            raise ValueError(" The embedding id cannot be bigger than input_dim. id = %d is not in [0, %d)"
                             % (mx, self.input_dim))

    def _gather_embedding_vectors(self, unique_ids):
        self._check_id_valid(unique_ids)
        if self._lookup_embedding_func is None:
            raise RuntimeError("Embedding layer %s has no lookup function; call "
                               "set_lookup_embedding_func(ps_client.pull_embedding_vectors)" % self._name)
        # the delegate passes its own name = the layer's embedding weight name (embedding.py:75-77)
        bet = self._lookup_embedding_func(self.embedding_weight_name, unique_ids)
        if not isinstance(bet, torch.Tensor):
            bet = torch.as_tensor(bet, dtype=torch.float32, device=unique_ids.device)
        return bet

    def _unique_and_pull(self, flat_ids, dropped=None):
        uniq, inv, n = ops.unique(flat_ids, 1)
        u = int(n.item())  # exact BET shape, as the reference exposes it
        if dropped is not None and int(dropped.item()):  # the stream is idle after n.item(): a 4-byte copy
            raise ValueError("sparse input has %d entries whose row index is outside [0, batch_size)"
                             % int(dropped.item()))
        unique_ids = uniq[:u]
        bet = self._gather_embedding_vectors(unique_ids)
        if self.tape:
            bet = bet.detach().requires_grad_(True)
            self._embedding_and_ids.append(EmbeddingAndIds(bet, unique_ids))
        return bet, inv

    def forward(self, ids):
        self._inputs_seen.append(ids)
        if self._prefetched is not None and self._prefetched[0] is ids:
            rows = self._prefetched[1]  # looked up with every other layer of the model before the forward pass
            self._prefetched = None
            return rows.reshape(tuple(ids.shape) + (self.output_dim,))
        if isinstance(ids, torch.Tensor) and ids.is_sparse:
            return self._sparse_input_call(ids)
        ids = torch.as_tensor(ids)
        if not ids.is_cuda:
            raise RuntimeError("Embedding input must live on the GPU (no CPU path)")
        ids = ids.to(torch.int64)
        flat_ids = ids.reshape(-1)
        k = flat_ids.numel()
        bet, inv = self._unique_and_pull(flat_ids)
        result = ops.GatherRows.apply(bet, inv, 1, k, self.output_dim)
        return result.reshape(tuple(ids.shape) + (self.output_dim,))

    call = forward

    def _sparse_input_call(self, sparse_input):
        if self.combiner not in ["sum", "mean", "sqrtn"]:
            raise ValueError("combiner must set sum, mean or sqrtn for sparse input")
        return self.safe_embedding_lookup_sparse(sparse_input, combiner=self.combiner)

    def safe_embedding_lookup_sparse(self, sparse_ids, combiner="mean"):
        """embedding_delegate.py:108-230 without weights: prune ids < 0, give empty rows
        id 0, combine per row, then zero the rows that were empty (ops.sparse_prep and
        ops.SparseCombine: CUDA kernels from the coalesced COO to the [batch, dim] output)."""
        sp = sparse_ids.coalesce()
        batch = sp.shape[0]
        nnz = sp.values().numel()
        ids, ws = ops.sparse_prep(sp.indices()[0], sp.values(), batch, self.output_dim)
        bet, inv = self._unique_and_pull(ids, dropped=ws[:4].view(torch.int32))
        return ops.SparseCombine.apply(bet, inv, ws, batch, nnz, combiner, self.output_dim)
