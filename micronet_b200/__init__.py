"""micronet_b200 — an H100 (sm_90a) engine for the fake-quant conv/linear hot path of
666DZY666/micronet, behind the reference's own module surface:

    from micronet_b200 import wbwtab, dorefa, iao     # <-> micronet.compression.quantization.{...}.quantize
    model = wbwtab.prepare(model, A=2, W=3)            # same prepare() rules and signatures

All arithmetic runs in hand-written CUDA kernels exported through the C-ABI in
``include/micronet_b200.h`` (``micronet_b200/lib/libmicronet_b200.so``); there is no CPU path."""
from . import _lib, functional  # noqa: F401
from . import bn_fuse, dorefa, fused, iao, wbwtab  # noqa: F401
from .parallel import FlatAdam, FlatGradBucket  # noqa: F401

__version__ = "0.1.0"
