"""Non-uniform k-means weight quantization (pytorch_quantizer/quantization/kmeans_quantization.py) on the GPU.

Every parameter that ``is_ignored`` lets through is clustered on its own with scikit-learn 1.9's 1-D
``KMeans(n_clusters=2**num_bits, random_state=0)`` (``ops.kmeans1d``: k-means++ and Lloyd in one launch of
csrc/fq_kmeans.cuh) and replaced by its cluster centres (task 'quantize') or clipped to [min, max] of the centres (task
'clip').  ``process_model`` saves the model, then the model with the per-output-channel bias correction.

    python cnn-quantization_b200/kmeans_quantization.py -a resnet18 -bits 4 -t quantize

The reference's names and arguments are kept; ``n_jobs`` is accepted and ignored.  The model is the seeded random-init
torchvision model (no pretrained weights are available offline).  Evaluate a saved model through the manager with
``qweight='f32'`` (INTEGRATION.md).
"""
import argparse
import copy
import os

import torch

try:
    from . import ops
    from .manager import search_absorbe_bn
except ImportError:   # run as a script
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.manager import search_absorbe_bn

SEED = 0   # the reference's KMeans(random_state=0)


def _as_cuda(x):
    t = torch.as_tensor(x)
    return (t if t.is_cuda else t.cuda()).float()


def clip1d_kmeans(x, num_bits=8, n_jobs=-1):
    """x clipped to [min, max] of its 2**num_bits 1-D k-means centres (kmeans_quantization.py:14-20).  A CUDA tensor
    (or anything torch.as_tensor takes, moved to the GPU); returns a CUDA tensor of x's shape."""
    t = _as_cuda(x)
    return ops.kmeans1d(t, num_bits, seed=SEED, task="clip").out


def quantize1d_kmeans(x, num_bits=8, n_jobs=-1):
    """Every value of x replaced by its 1-D k-means centre, 2**num_bits clusters (kmeans_quantization.py:23-30)."""
    t = _as_cuda(x)
    return ops.kmeans1d(t, num_bits, seed=SEED, task="quantize").out


def is_ignored(name, param):
    """The reference's rule (kmeans_quantization.py:33-39): the 1000-way 'fc' classifier, first-layer weights (3 input
    channels), biases, Inception's auxiliary head and its Conv2d_2a_3x3 weight."""
    return ('fc' in name and param.shape[0] == 1000) or \
           ('weight' in name and param.shape[1] == 3) or \
           ('bias' in name) or \
           ('AuxLogits' in name) or \
           (name == 'Conv2d_2a_3x3.conv.weight')


def _process_parameters(model, num_bits, task, rows=False):
    """Cluster every parameter is_ignored lets through in place; with ``rows`` also return {name: bias-corrected
    tensor} (kmeans_quantization.py:78-88)."""
    corrected = {}
    for name, p in model.named_parameters():
        if is_ignored(name, p):
            continue
        w = p.data if p.is_cuda else p.data.cuda()
        r = ops.kmeans1d(w, num_bits, seed=SEED, task=task, rows=w.shape[0] if rows else None)
        p.data = r.out.to(p.device).view(p.shape)
        if rows:
            corrected[name] = r.out_bcorr.to(p.device).view(p.shape)
    return corrected


def quantize_model_parameters(model, num_bits):
    """Quantize the parameters of the model with k-means (kmeans_quantization.py:42-46)."""
    _process_parameters(model, num_bits, "quantize")


def clip_model_parameters(model, num_bits):
    """Clip the parameters of the model to their k-means range (kmeans_quantization.py:49-53)."""
    _process_parameters(model, num_bits, "clip")


def model_paths(arch, num_bits, base_dir):
    """(quantized model, bias-corrected model) file names of process_model.  The reference derives the second with
    path.split('.')[0], which cuts at the first dot anywhere in the path (a dotted directory); here the extension is
    replaced instead."""
    path = os.path.join(base_dir, "models", arch + ("_kmeans%dbit.pt" % num_bits))
    return path, os.path.splitext(path)[0] + "_bcorr.pt"


def build_model(arch, seed=12345, device="cuda"):
    """The seeded random-init torchvision model with its BNs folded (kmeans_quantization.py:57-58)."""
    import torchvision.models as models
    torch.manual_seed(seed)
    model = models.__dict__[arch](weights=None)
    search_absorbe_bn(model)
    return model.to(device)


def process_model(arch, num_bits, base_dir, task="quantize", seed=12345, device="cuda"):
    """kmeans_quantization.py:56-92: cluster the model's parameters, save it, then save it with the per-output-channel bias
    correction w_q - (mean_row(w_q) - mean_row(w)).  Returns the two paths."""
    if task not in ("quantize", "clip"):
        raise ValueError("Invalid argument task=%s" % task)
    model = build_model(arch, seed, device)
    model_q = copy.deepcopy(model)
    corrected = _process_parameters(model_q, num_bits, task, rows=True)
    path, path_bcorr = model_paths(arch, num_bits, base_dir)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    print("Saving quantized model to %s" % path)
    torch.save(model_q, path)
    model_bcorr = copy.deepcopy(model_q)
    for name, p in model_bcorr.named_parameters():
        if name in corrected:
            p.data = corrected[name]
    print("Saving quantized model with bias correction to %s" % path_bcorr)
    torch.save(model_bcorr, path_bcorr)
    return path, path_bcorr


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('--arch', '-a', metavar='ARCH', default='resnet18')
    parser.add_argument('-bits', '--num_bits', default=4, type=int, help='Number of bits for quantization')
    parser.add_argument('-t', '--task', default='quantize', help='[quantize, clip]')
    parser.add_argument('--base-dir', default=os.path.join(os.path.expanduser("~"), 'mxt-sim'))
    args = parser.parse_args(argv)
    print('%s %s model to %d bits' % (args.task, args.arch, args.num_bits))
    process_model(args.arch, num_bits=args.num_bits, base_dir=args.base_dir, task=args.task)
    print('Done')


if __name__ == '__main__':
    main()
