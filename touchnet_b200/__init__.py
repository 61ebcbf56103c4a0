"""touchnet_b200 - H100-native (sm_90a) hot path of xingchensong/TouchNet (see DESIGN.md / INTEGRATION.md).

Importing the package does not load CUDA; the native library is loaded on first use and its absence is an error."""
__version__ = "0.1.0"

from . import _lib  # noqa: F401

__all__ = ["_lib", "ops", "modeling", "frontend", "batching", "loss", "tokenizer", "optim", "train_spec", "parallelize",
           "tensor_parallel", "context_parallel", "fsdp_comm", "generation"]
