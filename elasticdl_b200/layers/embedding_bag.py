"""nn.EmbeddingBag over the HBM parameter server: the pooled lookup of `Embedding`'s sparse input, taking the bag
input forms of torch.nn.EmbeddingBag (a [B, L] id tensor, or 1-D ids with offsets) instead of a COO tensor.

The ids go through ops.bag_prep (one launch: the filled id stream and the workspace ops.sparse_prep would give for the
equivalent COO), then the layer's unique + pull, then ops.SparseCombine, whose backward gives the [U, dim] rows the
trainer pushes.  Semantics are safe_embedding_lookup_sparse's (embedding_delegate.py:108-230): an empty bag (no kept
id) gives a zero row and puts the fill id 0 into the lookup; entries equal to `padding_idx` are dropped from the sum
and from the mean's count, as torch drops them; negative ids and bad offsets make the group's check() raise.
per_sample_weights (mode "sum" only, as in torch) weight each entry; a padding entry contributes nothing and gets
weight gradient 0.
"""
import torch

from elasticdl_b200 import ops
from elasticdl_b200.layers.embedding import Embedding

BAG_MODES = ("sum", "mean")


class EmbeddingBag(Embedding):
    """forward(input, offsets=None, per_sample_weights=None) -> [B, output_dim].  mode: "sum" or "mean" (the reference's combiners that torch
    shares; "max" has no reference counterpart)."""

    def __init__(self, output_dim, input_dim=None, mode="mean", embeddings_initializer="uniform",
                 include_last_offset=False, padding_idx=None, name=None):
        if mode not in BAG_MODES:
            raise ValueError("EmbeddingBag mode must be one of %s, not %r" % (BAG_MODES, mode))
        super().__init__(output_dim, input_dim=input_dim, embeddings_initializer=embeddings_initializer,
                         combiner=mode, name=name)
        self.mode = mode
        self.include_last_offset = bool(include_last_offset)
        self.padding_idx = None if padding_idx is None else int(padding_idx)
        self._group = None

    def set_ps_group(self, group):
        """The PSGroup whose error word reports bad offsets and negative ids (set by the trainer)."""
        self._group = group

    def prep(self, input, offsets=None):
        """(ids, ws, batch, nnz) of ops.bag_prep for this layer."""
        if self._group is None:
            raise RuntimeError("EmbeddingBag %s has no PS group; train it through ParameterServerTrainer" % self.name)
        return ops.bag_prep(self._group, input, offsets, self.output_dim, self.include_last_offset, self.padding_idx)

    def combine(self, bet, inv, ws, batch, nnz, per_sample_weights=None):
        return ops.SparseCombine.apply(bet, inv, ws, batch, nnz, self.mode, self.output_dim, per_sample_weights)

    def _check_weights(self, input, per_sample_weights):
        """torch.nn.functional.embedding_bag's rules: the shape of `input`, mode "sum" only."""
        if per_sample_weights is None:
            return None
        if input.size() != per_sample_weights.size():
            raise ValueError("embedding_bag: If per_sample_weights (%s) is not None, then it must have the same shape "
                             "as the input (%s)" % (per_sample_weights.shape, input.shape))
        if self.mode != "sum":
            raise NotImplementedError("embedding_bag: per_sample_weights was not None. per_sample_weights is only "
                                      "supported for mode='sum' (got mode='%s')" % self.mode)
        return per_sample_weights.reshape(-1).to(torch.float32)

    def forward(self, input, offsets=None, per_sample_weights=None):
        weights = self._check_weights(input, per_sample_weights)
        self._inputs_seen.append((input, offsets))
        pre = self._prefetched
        if pre is not None and pre[0] is input and pre[1] is offsets:
            self._prefetched = None  # prepared and looked up with the other layers before the forward pass
            return self.combine(*pre[2:], weights)
        ids, ws, batch, nnz = self.prep(input, offsets)
        bet, inv = self._unique_and_pull(ids)
        return self.combine(bet, inv, ws, batch, nnz, weights)

    call = forward
