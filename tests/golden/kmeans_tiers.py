"""Comparison rules of the k-means fixtures (kmeans_ref.npz, written by make_kmeans_golden.py from scikit-learn's runs of
the reference script), shared by the CPU tests of the restatement and the GPU tests of ops.kmeans1d.

Tier (i), started from scikit-learn's own init centres: the same n_iter, the sorted centres within TIER_I_CENTRES of the
data range, the sampled labels equal but for a fraction of TIER_I_LABELS.  scikit-learn runs the fit in float32 (per-chunk
float32 sums, float32 centring), the restatement in float64; over most tensors the centres agree to 1e-7 of the range
and the labels exactly.  The bounds are the measured worst cases with headroom: ResNet-18 layer2.0.conv2 (41 iterations,
the longest run) drifts to 2.1e-5 of the range with 3.2e-4 of its labels moved.  At 8 bits (mid_8bit: 256 clusters of
147456 values, 8 vs 9 iterations) the two arithmetics stop one iteration apart; that tensor is held to the inertia only, within
0.5 % (measured: 0.29 %).

Tier (ii), end to end: the first k-means++ pick is the same (it does not depend on the data); the later picks need not be
(scikit-learn's potentials are float32 BLAS dots), so the inertia is held within TIER_II_INERTIA relative, the largest
deviation measured over the fixtures being 5.1 % (ResNet-18 layer2.1.conv2).  The tensor of 9 distinct values has a zero
inertia up to rounding in both runs."""
import hashlib

import numpy as np

import kmeans_oracle as KO

TIER_I_CENTRES = 3e-5
TIER_I_LABELS = 5e-4
TIER_I_INERTIA_ONLY = {"synthetic/mid_8bit": 5e-3}
TIER_II_INERTIA = 0.06


def names(ref):
    return sorted(k[len("ref_centres/"):] for k in ref.files if k.startswith("ref_centres/"))


_MODEL = {}


def fixture_tensor(ref, name):
    """The input of fixture `name`, regenerated (seeded ResNet-18 weight or synthetic tensor) and checked by its SHA-1."""
    src, nm = name.split("/", 1)
    if src == "resnet18":
        if "resnet18" not in _MODEL:
            from cnn_quantization_b200 import kmeans_quantization as KQ
            _MODEL["resnet18"] = {n: p.detach().numpy().copy() for n, p in KQ.build_model("resnet18", device="cpu").named_parameters()}
        x = _MODEL["resnet18"][nm].reshape(-1)
    else:
        x = KO.synthetic(*KO.SYNTHETIC[nm][:3])
    x = np.ascontiguousarray(x, dtype=np.float32)
    assert hashlib.sha1(x.tobytes()).hexdigest() == str(ref["sha1/" + name]), "fixture input %s differs" % name
    return x


def check_tier_i(ref, name, x, n_iter, centres, labels, inertia):
    rng = float(x.max()) - float(x.min())
    if name in TIER_I_INERTIA_ONLY:
        ri = float(ref["ref_inertia/" + name])
        assert abs(inertia - ri) <= TIER_I_INERTIA_ONLY[name] * ri, (name, inertia / ri - 1)
        return
    assert n_iter == int(ref["ref_n_iter/" + name]), name
    dc = np.abs(np.sort(np.asarray(centres, np.float64)) - np.sort(ref["ref_centres/" + name])).max()
    assert dc <= TIER_I_CENTRES * rng, (name, dc / rng)
    bad = np.mean(np.asarray(labels)[KO.sample_positions(x.size)] != ref["ref_labels/" + name])
    assert bad <= TIER_I_LABELS, (name, bad)


def check_tier_ii(ref, name, x, init_ids, inertia):
    assert int(init_ids[0]) == int(ref["ref_init_ids/" + name][0]), name
    ri = float(ref["ref_inertia/" + name])
    rng = float(x.max()) - float(x.min())
    assert abs(inertia - ri) <= TIER_II_INERTIA * ri + 1e-9 * x.size * rng * rng, (name, inertia, ri)
