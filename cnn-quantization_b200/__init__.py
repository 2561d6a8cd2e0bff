"""cnn-quantization_b200: H100-native (sm_90a) implementation of the fake-quantization hot path of
submission2019/cnn-quantization, behind the reference's own ``int_quantization`` / ``IntQuantizer`` API.

    from cnn_quantization_b200 import int_quantization          # drop-in for the compiled extension module
    from cnn_quantization_b200.int_quantizer import IntQuantizer, int_quantizer

The arithmetic lives in ``libfqb200.so`` (C ABI: include/fqb200.h; CUDA sources: csrc/).  There is no CPU
implementation in this package: calling a compute entry point without the built library or with CPU tensors
raises.
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401
from . import ops  # noqa: F401
from . import int_quantization  # noqa: F401
from .dummy_quantizer import DummyQuantizer  # noqa: F401
from .int_quantizer import IntQuantizer, int_quantizer  # noqa: F401
