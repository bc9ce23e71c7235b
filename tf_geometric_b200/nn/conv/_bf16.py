# coding=utf-8
"""The bf16 message-row mode (message_dtype=torch.bfloat16) of the convolutions: inference in which every table that is
gathered along edges is stored in bf16, rounded once to nearest even, and aggregated in fp32 from half the bytes.  Self
terms, addends, accumulators, GEMM operands and outputs stay fp32; the arithmetic order is the fp32 path's."""
from ... import ops, autograd
from ...sparse import as_sparse_features


def enabled(message_dtype):
    """True for torch.bfloat16 / "bfloat16", False for None / torch.float32; ValueError for anything else."""
    return ops.message_dtype(message_dtype) is not None


def refuse_unsupported(x, operands=(), dropout=False):
    """The bf16 mode is inference over a dense x: NotImplementedError for a sparse x, for active dropout (`dropout`: a
    rate > 0 while training) and for any operand that requires grad."""
    if as_sparse_features(x) is not None:
        raise NotImplementedError("message_dtype=bfloat16 takes a dense x")
    if dropout:
        raise NotImplementedError("message_dtype=bfloat16 is for inference: dropout is not applied in bf16")
    if autograd.needs_grad(x, *operands):
        raise NotImplementedError("message_dtype=bfloat16 is for inference: no operand may require grad")
