"""TEST INFRASTRUCTURE (like everything under oracle/): the REFERENCE itself as a live oracle on the GPU box.

oracle/build_oracle.py stages the reference's Python packages unmodified under oracle/_ref/pyref and compiles its CUDA
extension unmodified into oracle/_ref/ (both git-ignored build products of build()).  This module imports
them so that GPU tests can run ``IntQuantizer`` (int_quantizer.py:56-632) and the reference's own inference manager
(inference_quantization_manager.py) on the very CUDA tensors our kernels see, at any size.

Only tests/, __graft_entry__.smoke() and bench.py's baseline legs may import this; the product never does.
"""
import glob
import importlib
import importlib.util
import os
import sys
import types
from itertools import count

HERE = os.path.dirname(os.path.abspath(__file__))
REFDIR = os.path.join(HERE, "_ref")
PYREF = os.path.join(REFDIR, "pyref")
_MARKER = os.path.join(PYREF, "pytorch_quantizer", "quantization", "qtypes", "int_quantizer.py")

_state = {}


def ext_path():
    from oracle.build_oracle import REF_EXT_DIR   # built for this project's GPU architecture, nothing else
    found = glob.glob(os.path.join(REF_EXT_DIR, "int_quantization*.so"))
    return found[0] if found else None


def available():
    """True when both the staged Python packages and the reference's compiled extension are present."""
    return os.path.exists(_MARKER) and ext_path() is not None


def python_available():
    """True when the reference's Python path is staged (enough for the CPU legs)."""
    return os.path.exists(_MARKER)


def load_extension():
    """The reference's own compiled ``int_quantization`` module (kernels/int_quantization.cpp + gemmlowp.cu)."""
    if "ext" not in _state:
        import torch  # noqa: F401  (the extension links against libtorch)
        spec = importlib.util.spec_from_file_location("int_quantization", ext_path())
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _state["ext"] = mod
    return _state["ext"]


def load(extension=None):
    """Import the staged reference.  ``extension`` is the module served as ``int_quantization`` (default: the
    reference's own compiled extension).  Returns a namespace with ``iq`` (the int_quantizer module), ``iqm`` (the
    inference manager module), ``IntQuantizer``, ``int_quantizer``, ``utils`` helpers."""
    if "ns" in _state:
        if extension is not None:
            set_extension(extension)
        return _state["ns"]
    if not os.path.exists(_MARKER):
        raise RuntimeError("oracle/_ref/pyref is not staged (run __graft_entry__.build() where /root/reference exists)")
    ext = extension if extension is not None else load_extension()
    saved = sys.modules.get("int_quantization")
    sys.modules["int_quantization"] = ext
    for name in ("mlflow", "tensorboardX", "bokeh"):  # imported by utils/mllog.py / utils/log.py, never used on the path
        sys.modules.setdefault(name, types.ModuleType(name))
    if PYREF not in sys.path:
        sys.path.insert(0, PYREF)
    try:
        iq = importlib.import_module("pytorch_quantizer.quantization.qtypes.int_quantizer")
        iqm = importlib.import_module("pytorch_quantizer.quantization.inference.inference_quantization_manager")
        absorb = importlib.import_module("utils.absorb_bn")
        mark = importlib.import_module("utils.mark_relu")
        naming = importlib.import_module("utils.model_naming")
        misc = importlib.import_module("utils.misc")
        qtypes = importlib.import_module("pytorch_quantizer.quantization.qtypes")
    finally:
        if saved is not None:
            sys.modules["int_quantization"] = saved
        else:
            sys.modules.pop("int_quantization", None)
    ns = types.SimpleNamespace(iq=iq, iqm=iqm, IntQuantizer=iq.IntQuantizer, int_quantizer=iq.int_quantizer,
                               search_absorbe_bn=absorb.search_absorbe_bn,
                               resnet_mark_before_relu=mark.resnet_mark_before_relu,
                               set_node_names=naming.set_node_names, Singleton=misc.Singleton, qtypes=qtypes,
                               reference_factory=iq.int_quantizer)
    _state["ns"] = ns
    return ns


def set_extension(module):
    """Rebind the module the already-imported reference calls as ``int_quantization`` (int_quantizer.py:4,
    clipping_manager.py:4)."""
    ns = _state["ns"]
    ns.iq.int_quantization = module
    cm = sys.modules.get("pytorch_quantizer.clipping.clipping_manager")
    if cm is not None:
        cm.int_quantization = module


def set_quantizer_factory(factory=None):
    """What ``TruncationOpManagerInference.__load_quantizer__`` resolves (inference_quantization_manager.py:401-405):
    ``None`` restores the reference's own ``int_quantizer``."""
    ns = _state["ns"]
    ns.qtypes.int_quantizer = factory if factory is not None else ns.reference_factory


class LeafSpy(object):
    """Records what the reference's leaves receive: (delta, offset, bit_alloc) of ``__gemmlowpQuantize1__`` and
    (delta, offset) of ``__gemmlowpQuantize__``."""

    def __init__(self, quantizer):
        self.q = quantizer
        self.calls = []

    def __enter__(self):
        q, calls = self.q, self.calls
        self._o1 = q.__gemmlowpQuantize1__
        self._o0 = q.__gemmlowpQuantize__

        def leaf1(tensor, delta, offset, bit_alloc=None, measure_entropy=False):
            calls.append(("torch", delta.detach().clone() if hasattr(delta, "detach") else delta,
                          offset.detach().clone() if hasattr(offset, "detach") else offset,
                          None if bit_alloc is None else bit_alloc.detach().clone()))
            return self._o1(tensor, delta, offset, bit_alloc=bit_alloc, measure_entropy=measure_entropy)

        def leaf0(tensor, delta, offset):
            calls.append(("compiled", delta, offset, None))
            return self._o0(tensor, delta, offset)

        q.__gemmlowpQuantize1__ = leaf1
        q.__gemmlowpQuantize__ = leaf0
        return self

    def __exit__(self, *exc):
        del self.q.__dict__["__gemmlowpQuantize1__"]
        del self.q.__dict__["__gemmlowpQuantize__"]


def cpu_extension():
    """Stand-in for the compiled ``int_quantization`` module on hosts without a GPU: the oracle's plain-C restatement of
    kernels/gemmlowp.cu (oracle/fq_leaf.c).  Used by the CPU legs of bench.py and by the fixture generators."""
    from oracle import fq_oracle as O
    stub = types.ModuleType("int_quantization")
    stub.float2gemmlowp = lambda t, d, o, b, ie, tz, noise: O.float2gemmlowp(t, float(d), float(o), b, ie, tz, None)
    return stub


class cpu_mode(object):
    """Run the staged reference on CPU tensors: ``IntQuantizer.__gemmlowpQuantize__`` allocates its noise tensor with
    ``torch.cuda.FloatTensor`` (int_quantizer.py:610) and utils/absorb_bn.py:19-20 hard-codes ``.cuda()``; inside this
    context the former goes to the C restatement of the kernel (same preserve_zero rule) and the latter is a no-op when no
    GPU is present.  Every other executed line is the reference's."""

    def __enter__(self):
        import torch
        ns = load(extension=cpu_extension()) if "ns" not in _state else _state["ns"]
        set_extension(cpu_extension())
        self._orig_leaf = ns.IntQuantizer.__gemmlowpQuantize__
        ext = ns.iq.int_quantization

        def leaf_cpu(q, tensor, delta, offset):
            preserve_zero = q.enforce_true_zero and (offset + delta) > 0 and offset < 0
            return ext.float2gemmlowp(tensor.contiguous(), delta, offset, q.num_bits, q.int_exp, bool(preserve_zero), None)

        ns.IntQuantizer.__gemmlowpQuantize__ = leaf_cpu
        self._orig_cuda = torch.Tensor.cuda
        if not torch.cuda.is_available():
            torch.Tensor.cuda = lambda t, *a, **k: t
        return ns

    def __exit__(self, *exc):
        import torch
        ns = _state["ns"]
        ns.IntQuantizer.__gemmlowpQuantize__ = self._orig_leaf
        torch.Tensor.cuda = self._orig_cuda
        if ext_path() is not None and torch.cuda.is_available():
            set_extension(load_extension())


def reset_reference_singletons():
    ns = _state["ns"]
    ns.Singleton._instances.clear()
    for cls in (ns.iqm.Conv2dWithId, ns.iqm.LinearWithId, ns.iqm.MaxPool2dWithId, ns.iqm.AvgPool2dWithId,
                ns.iqm.BatchNorm2dWithId):
        cls._id = count(0)


def build_reference_model(args, qparams, device, seed=12345, channels_last=False):
    """The model exactly as inference_sim.py:131-229 prepares it, driven by the REFERENCE's manager (class swap,
    quantize_model).  Returns (model, manager); the manager stays entered - call ``manager.__exit__()`` when done."""
    import torch
    import torchvision.models as models
    ns = load()
    reset_reference_singletons()
    qm = ns.iqm.QuantizationManagerInference(args, qparams)
    qm.__enter__()
    try:
        torch.manual_seed(seed)  # inference_sim.py:127
        model = models.__dict__[args.arch](weights=None)
        ns.set_node_names(model)
        if "resnet" in args.arch:
            ns.resnet_mark_before_relu(model)
        if "resnet" in args.arch or args.arch in ("vgg16_bn", "inception_v3"):
            ns.search_absorbe_bn(model)  # on the CPU copy, like inference_sim.py:187-190 (its buffers go .cuda())
            qm.bn_folding = True
        model.eval()
        model = model.to(device)
        if channels_last:
            model = model.to(memory_format=torch.channels_last)
        qm.quantize_model(model)
    except Exception:
        qm.__exit__()
        raise
    return model, qm
