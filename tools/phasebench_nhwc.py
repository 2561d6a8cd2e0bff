"""Phase-boundary timestamps of the fused kernels, NCHW next to channels-last (diagnostic tool; fqb200_desc.debug_stamps,
%globaltimer, us).  Usage: python tools/phasebench_nhwc.py [N C HW ...]"""
import sys
import torch
sys.path.insert(0, ".")
import cnn_quantization_b200 as fq
from cnn_quantization_b200 import _lib as L
buf = torch.zeros(16, dtype=torch.int64, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
order = [(0, "start"), (13, "S1 streamed"), (2, "comb min"), (3, "comb max"), (6, "comb S"), (1, "S1 combined"), (4, "past barrier 1"),
         (10, "aux: std"), (15, "aux: pow+sum"), (11, "aux: iterations"), (12, "aux solved"), (14, "S2 streamed"), (5, "S2 combined"), (7, "params ready"), (8, "past barrier 2"),
         (9, "apply done")]
shapes = [(512, 64, 56), (512, 256, 14), (512, 128, 28), (512, 1024, 14), (512, 2048, 7), (512, 512, 7), (512, 512, 14),
          (128, 64, 56), (128, 256, 14), (128, 512, 7), (128, 1024, 14), (128, 256, 56)]
cl_only = "--cl-only" in sys.argv
sys.argv = [a for a in sys.argv if a != "--cl-only"]
if len(sys.argv) > 3:
    v = [int(a) for a in sys.argv[1:]]
    shapes = [tuple(v[i:i + 3]) for i in range(0, len(v), 3)]
for (n, c, hw) in shapes:
    for cl in ((True,) if cl_only else (False, True)):
        x = torch.randn(n, c, hw, hw, device="cuda")
        if cl:
            x = x.contiguous(memory_format=torch.channels_last)
        lay = (n, c, hw * hw)
        best = None
        for rep in range(4):
            flush.zero_()
            buf.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fq.ops.fused(x, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True, out=x, channels_last=cl, debug_stamps=buf)
            e.record()
            torch.cuda.synchronize()
            tot = s.elapsed_time(e) * 1e3
            if rep and (best is None or tot < best[0]):
                best = (tot, buf.cpu().tolist())
        tot, t = best
        gb = n * c * hw * hw * 16 / 1e9
        print((n, c, hw), "NHWC" if cl else "NCHW", "total %.1f us (%.2f of the H100 data sheet's 3350 GB/s)" % (tot, gb / (tot * 1e-6) / 3350.0),
              " | ".join("%s %.1f" % (nm, (t[i] - t[0]) / 1e3) for i, nm in order if t[i]))
