#!/usr/bin/env python
"""k-means fixtures from the REAL reference script (build container only; needs the reference checkout and scikit-learn):

    python tests/golden/make_kmeans_golden.py  ->  tests/golden/kmeans_ref.npz

Runs the reference's own process_model (pytorch_quantizer/quantization/kmeans_quantization.py:56-92, quantize task, 4 bits)
on the seeded, BN-folded ResNet-18 (torch.manual_seed(12345), random init: the torchvision constructor is swapped for one
that ignores pretrained=True), and its quantize1d_kmeans / clip1d_kmeans on the synthetic tensors of kmeans_oracle.py.
In this process only:
- sys.argv is set before the import (the module parses it at import time);
- torch.Tensor.cuda is the identity (utils/absorb_bn.py:19-20 hard-codes .cuda(), as make_census.py does);
- the module's KMeans is a subclass that drops n_jobs (scikit-learn >= 1.0 rejects it) and records, per fit, the init
  centres (what _init_centroids returns: the data points X[ids] centred in float32; stored as the data values x[ids]),
  the k-means++ sample indices,
  n_iter_, inertia_, cluster_centers_ and labels_.
Per tensor the file keeps: a SHA-1 of the input, the centres, the init centres and indices, n_iter, inertia, the label
counts, the labels at kmeans_oracle.sample_positions, the clip bounds; the reference's bias-corrected layer1.0.conv1.weight;
and is_ignored's decisions over the BN-folded ResNet-50, VGG-16 and Inception-v3 parameter names.
"""
import hashlib
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, "/root/reference")
import kmeans_oracle as KO  # noqa: E402

sys.argv = ["kmeans_quantization.py"]
torch.Tensor.cuda = lambda self, *a, **k: self
import sklearn.cluster._kmeans as skk  # noqa: E402
import torchvision.models as tvm  # noqa: E402
from pytorch_quantizer.quantization import kmeans_quantization as ref  # noqa: E402

LAST = {}
_kpp = skk._kmeans_plusplus


def _kpp_rec(*a, **k):
    centres, ids = _kpp(*a, **k)
    LAST["init_ids"] = np.asarray(ids).copy()
    return centres, ids


skk._kmeans_plusplus = _kpp_rec


class RecKMeans(skk.KMeans):
    def __init__(self, n_clusters=8, random_state=None, n_jobs=None):
        super().__init__(n_clusters=n_clusters, random_state=random_state)
        self.n_jobs = n_jobs

    def _init_centroids(self, *a, **k):
        c = super()._init_centroids(*a, **k)
        LAST["init"] = np.asarray(c)[:, 0].copy()
        return c

    def fit(self, X, y=None, sample_weight=None):
        X32 = np.asarray(X, dtype=np.float32)
        mean = X32.mean(axis=0)
        super().fit(X, y, sample_weight)
        # k-means++ picks data points: the init centres are X[ids] centred in float32; keep the data values themselves
        ids = LAST["init_ids"]
        assert np.array_equal(LAST["init"], X32[ids, 0] - mean[0])
        LAST.update(init=X32[ids, 0].astype(np.float64), n_iter=self.n_iter_,
                    inertia=self.inertia_, centres=self.cluster_centers_[:, 0].astype(np.float64),
                    labels=self.labels_.copy(), x=X32[:, 0].copy())
        RECORDS.append(dict(LAST))
        return self


ref.KMeans = RecKMeans
RECORDS = []


def seeded(arch):
    torch.manual_seed(12345)
    return tvm.__dict__[arch](weights=None)


def record(out, name, rec, bits, clip=None):
    x = rec["x"]
    pos = KO.sample_positions(x.size)
    out["sha1/" + name] = np.array(hashlib.sha1(x.tobytes()).hexdigest())
    out["bits/" + name] = np.array(bits)
    out["ref_centres/" + name] = rec["centres"]
    out["ref_init/" + name] = rec["init"]
    out["ref_init_ids/" + name] = np.asarray(rec["init_ids"], dtype=np.int64)
    out["ref_n_iter/" + name] = np.array(rec["n_iter"])
    out["ref_inertia/" + name] = np.array(rec["inertia"])
    out["ref_counts/" + name] = np.bincount(rec["labels"], minlength=1 << bits)
    out["ref_labels/" + name] = rec["labels"][pos].astype(np.uint8)
    if clip is not None:
        out["ref_clip/" + name] = np.array([clip.min(), clip.max()], dtype=np.float64)


def main():
    out = {}
    # ResNet-18 through the reference's process_model (quantize, 4 bits)
    ref.models = types.SimpleNamespace(resnet18=lambda pretrained=True: seeded("resnet18"))
    base = tempfile.mkdtemp()
    RECORDS.clear()
    ref.process_model("resnet18", num_bits=4, base_dir=base, task="quantize")
    model = seeded("resnet18")
    ref.search_absorbe_bn(model)
    names = [n for n, p in model.named_parameters() if not ref.is_ignored(n, p)]
    assert len(names) == len(RECORDS)
    for name, rec in zip(names, RECORDS):
        record(out, "resnet18/" + name, rec, 4)
    bc = torch.load(os.path.join(base, "models", "resnet18_kmeans4bit_bcorr.pt"), weights_only=False)
    out["ref_bcorr/resnet18/layer1.0.conv1.weight"] = dict(bc.named_parameters())["layer1.0.conv1.weight"].detach().numpy().reshape(-1)
    out["saved"] = np.array(sorted(os.listdir(os.path.join(base, "models"))))
    # synthetic tensors through quantize1d_kmeans and clip1d_kmeans
    for name, (kind, n, seed, bits) in KO.SYNTHETIC.items():
        x = KO.synthetic(kind, n, seed)
        RECORDS.clear()
        ref.quantize1d_kmeans(x, num_bits=bits)
        clip = ref.clip1d_kmeans(x, num_bits=bits)
        record(out, "synthetic/" + name, RECORDS[0], bits, clip)
    # is_ignored over BN-folded models
    for arch in ("resnet50", "vgg16", "inception_v3"):
        m = tvm.__dict__[arch](weights=None, init_weights=False) if arch == "inception_v3" else seeded(arch)
        ref.search_absorbe_bn(m)
        ps = list(m.named_parameters())
        out["ignored_names/" + arch] = np.array([n for n, _ in ps])
        out["ignored_shapes/" + arch] = np.array([list(p.shape) + [0] * (4 - p.dim()) for _, p in ps], dtype=np.int64)
        out["ignored/" + arch] = np.array([ref.is_ignored(n, p) for n, p in ps])
    np.savez_compressed(os.path.join(HERE, "kmeans_ref.npz"), **out)


if __name__ == "__main__":
    main()
