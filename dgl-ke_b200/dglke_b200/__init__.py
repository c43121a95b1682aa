"""dglke_b200 -- host-side mirror of awslabs/dgl-ke's training plugin surface
(KEModel / score_func / ExternalEmbedding / LossGenerator / dglke_train flags) on top of
libkge_b200.so, the hand-written sm_90a implementation of the per-step hot path.

PyTorch is used for device memory, streams and torch.distributed only; all arithmetic of the
step runs in the CUDA library.  There is no CPU or eager-PyTorch fallback."""
__version__ = "0.1.0"

from ._lib import KgeError, LIB_PATH, load_library, get_handle  # noqa: F401
