"""tinychatengine_b200 -- H100 (sm_90a) implementation of TinyChatEngine's quantized-linear hot path.

The product is ``lib/libtce_b200.so`` (hand-written CUDA behind the C ABI in ``include/tce_b200.h``); this
package is the thin host layer: the ctypes binding (:mod:`._lib`), the reference's on-disk INT4 formats
(:mod:`.formats`), Python mirrors of the reference's op classes (:mod:`.ops`) and the Llama decode runner
(:mod:`.llama`).  PyTorch is used for device memory, streams and torch.distributed only.

There is no CPU fallback: importing works anywhere, any compute call without the CUDA library / a GPU raises.
"""
from .build import build  # noqa: F401

__all__ = ["build"]
