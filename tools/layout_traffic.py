"""DRAM traffic per element of the fused channels-last launch, one launch per distinct ResNet-50 / ResNet-101 layout
(diagnostic; round-1 VERDICT item 3 asked for the DRAM bytes of the L2-resident layouts).

    ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none \
        -k regex:fq_cl_kernel --csv --log-file layout_traffic.csv python tools/layout_traffic.py
    python tools/layout_traffic.py --summarise layout_traffic.csv

Every launch runs on a tensor a 256 MB memset has just pushed out of L2 (the worst case: inside a model step the
convolution that produced the tensor leaves part of it in L2)."""
import csv
import sys

SHAPES = [(512, 64, 112), (512, 256, 56), (512, 64, 56), (512, 128, 56), (512, 512, 28), (512, 128, 28), (512, 256, 28),
          (512, 1024, 14), (512, 256, 14), (512, 512, 14), (512, 2048, 7), (512, 512, 7),
          (128, 256, 56), (128, 64, 56), (128, 512, 28), (128, 128, 28), (128, 1024, 14), (128, 256, 14), (128, 2048, 7),
          (128, 512, 7)]

if "--summarise" in sys.argv:
    path = sys.argv[sys.argv.index("--summarise") + 1]
    rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) >= 15 and r[0].isdigit()]
    launches = {}
    for r in rows:
        m = launches.setdefault(int(r[0]), {})
        v = float(r[14].replace(",", ""))
        unit = r[13]
        scale = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "usecond": 1e-6, "us": 1e-6, "nsecond": 1e-9, "ns": 1e-9,
                 "msecond": 1e-3, "ms": 1e-3}.get(unit, 1.0)
        m[r[12]] = v * scale
    ids = sorted(launches)
    assert len(ids) == len(SHAPES), (len(ids), len(SHAPES))
    print("%-16s %10s %9s %9s %9s %9s" % ("layout (NHWC)", "MB", "us (ncu)", "read B/el", "write B/el", "total B/el"))
    for lid, (n, c, hw) in zip(ids, SHAPES):
        m = launches[lid]
        el = n * c * hw * hw
        rd, wr = m["dram__bytes_read.sum"] / el, m["dram__bytes_write.sum"] / el
        print("%-16s %10.1f %9.1f %9.2f %9.2f %9.2f" % ("%dx%dx%dx%d" % (n, c, hw, hw), el * 4 / 1e6,
                                                        m["gpu__time_duration.sum"] * 1e6, rd, wr, rd + wr))
    sys.exit(0)

import torch
sys.path.insert(0, ".")
import cnn_quantization_b200 as fq
from cnn_quantization_b200 import _lib as L

flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for (n, c, hw) in SHAPES:
    x = torch.randn(n, c, hw, hw, device="cuda").contiguous(memory_format=torch.channels_last)
    flush.zero_()
    fq.ops.fused(x, (n, c, hw * hw), range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True, out=x, channels_last=True)
    torch.cuda.synchronize()
    del x
