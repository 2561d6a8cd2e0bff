#!/usr/bin/env python
"""bench.py - inference throughput of a BASELINE.json configuration through the fused sm_90a fake-quantization path.

    python bench.py --gpus N --steps K --warmup W            # this framework (one rank per GPU under torchrun)
    python bench.py ... --dump-outputs DIR                   # + what the last timed step computed, as DIR/<name>.npy
    python bench.py --impl reference --gpus N --steps K ...  # the reference's own Python on the box's host CPU cores

Default workload = BASELINE.json configs[2]: ResNet-50 W4A4 (-pcq_w -pcq_a -c laplace -baa -baw -bcw), batch 512 per GPU,
synthetic 3x224x224 input, random-init torchvision weights.  A step = one forward of the hooked model over one batch
(55 hooked activation tensors, 5.79 G elements).  Prints ONE JSON line (rank 0).  DESIGN.md "Measurement" explains every
key; the other BASELINE configs ride along as secondary results (`--no-secondary` skips them).
"""
import argparse
import contextlib
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

UNIT = "images/s"

# --config -> (BASELINE.json configs index, reference CLI flags for the workload string)
WORKLOADS = {
    "resnet50_w8a8": (1, "--qtype int8"),
    "resnet50_w4a4": (2, "-pcq_w -pcq_a -c laplace -baa -baw -bcw"),
    "resnet101_w4a4": (3, "-pcq_w -pcq_a -c laplace -baa -baw -bcw"),
    "vgg16_w4a4": (4, "-pcq_w -pcq_a -c laplace -baa -baw -bcw -bata 5.3 -batw 5.3"),
    "vgg16_w4a4_mtq": (4, "-pcq_w -pcq_a -c laplace -baa -baw -bcw -bata 5.3 -batw 5.3 -mtq"),
    "resnet18_w4a4": (2, "-pcq_w -pcq_a -c laplace -baa -baw -bcw (ResNet-18)"),
}

# DRAM traffic of the dominant kernel, from profiles/ncu_traffic.json when present (bench.py cannot run under ncu itself):
# ncu dram__bytes_read.sum + dram__bytes_write.sum averaged over the mode-D launches of one step of the named workload.
NCU_TRAFFIC_BYTES_PER_LAUNCH = {}
try:
    with open(os.path.join(ROOT, "profiles", "ncu_traffic.json")) as _f:
        for _k, _v in json.load(_f).items():
            NCU_TRAFFIC_BYTES_PER_LAUNCH[_k] = (_v["bytes_per_launch"], _v["source"])
except (OSError, ValueError, KeyError):
    pass


def metric_name(config):
    return "%s_images_per_s" % config


def workload_string(config, batch):
    idx, flags = WORKLOADS.get(config, (None, ""))
    return "BASELINE configs[%s]: %s (%s), batch %d per GPU, 3x224x224, random-init torchvision weights" % (
        idx, config, flags, batch)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="fqb200", choices=["fqb200", "reference"])
    ap.add_argument("--config", default="resnet50_w4a4", choices=sorted(WORKLOADS))
    ap.add_argument("--batch", type=int, default=512, help="images per GPU per step")
    ap.add_argument("--cpu-batch", type=int, default=32, help="images per step of the CPU reference arm / cpu_baseline")
    ap.add_argument("--cpu-budget-s", type=float, default=240.0, help="wall-clock cap of the CPU reference arm")
    ap.add_argument("--nchw", action="store_true",
                    help="keep the model's tensors in contiguous NCHW memory (fq_fused_kernel) instead of the default "
                         "torch.channels_last memory format (fq_cl_kernel, no cuDNN layout conversions)")
    ap.add_argument("--channels-last", action="store_true", help="accepted for compatibility: this is the default")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true", help="skip the other BASELINE configs, kernel_bench and gpu_baseline")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (rank 0) as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    args.channels_last = not args.nchw
    return args


def peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            p = json.load(f)
        return float(p["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, "H100 SXM data sheet (HBM3, 3.35 TB/s)"


class ClockSampler(object):
    """SM clock, power and throttle reasons sampled through NVML every 100 ms while the timed region runs."""

    def __init__(self, index):
        self.index, self.rows, self.stop_flag, self.thread, self.err = index, [], threading.Event(), None, None

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(self.index)
            self.max_sm = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception as e:  # pragma: no cover
            self.err = repr(e)
            return
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def _run(self):
        nv = self.nv
        while not self.stop_flag.is_set():
            try:
                sm = nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)
                pw = nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0
                rs = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                self.rows.append((sm, pw, rs))
            except Exception as e:  # pragma: no cover
                self.err = repr(e)
                return
            time.sleep(0.1)

    def stop(self):
        if self.thread is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvml unavailable: %s" % self.err]}
        self.stop_flag.set()
        self.thread.join(timeout=2)
        nv = self.nv
        names = {"hw_slowdown": nv.nvmlClocksEventReasonHwSlowdown, "hw_thermal_slowdown": nv.nvmlClocksEventReasonHwThermalSlowdown,
                 "sw_thermal_slowdown": nv.nvmlClocksEventReasonSwThermalSlowdown, "sw_power_cap": nv.nvmlClocksEventReasonSwPowerCap}
        seen = set()
        for _, _, rs in self.rows:
            for k, bit in names.items():
                if rs & bit:
                    seen.add(k)
        busy = sorted(sm for sm, pw, _ in self.rows if pw > 250.0) or sorted(sm for sm, _, _ in self.rows)
        return {"sm_mhz": busy[len(busy) // 2] if busy else None, "sm_max_mhz": self.max_sm, "samples": len(self.rows),
                "power_w_max": max((pw for _, pw, _ in self.rows), default=None), "reasons": sorted(seen)}


# ---------------------------------------------------------------------------------------------------
# CPU legs: the reference's own Python (staged under oracle/_ref/pyref by build()), else the oracle port
# ---------------------------------------------------------------------------------------------------
def _cpu_threads():
    import torch
    from oracle.host import host_threads
    cores = host_threads()
    torch.set_num_threads(cores)
    return cores


def cpu_pipeline(config, batch, steps, warmup, budget_s):
    """The hooked model on the host cores.  Returns a dict: images/s, seconds per step, threads, steps done, kind
    ('reference': the staged reference manager + IntQuantizer; 'port': this repo's manager + the oracle port), and the
    share of a step spent inside quantize_instant (the hot path; the rest is torch CPU convolutions)."""
    import torch
    from cnn_quantization_b200 import manager as M, pipeline
    from oracle import ref_live
    cores = _cpu_threads()
    flags = dict(pipeline.CONFIGS[config])
    x, t = pipeline.synthetic_batch(batch, seed=1)
    quant_s = [0.0]

    def timed(fn):
        def wrapper(*a, **k):
            t0 = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                quant_s[0] += time.perf_counter() - t0
        return wrapper

    if ref_live.python_available():
        kind = "reference"
        ctx = ref_live.cpu_mode()
        ns = ctx.__enter__()
        args = M.make_args(**flags)
        with contextlib.redirect_stdout(sys.stderr):
            model, qm = ref_live.build_reference_model(args, M.get_params(args), "cpu")
        cls = ns.iqm.TruncationOpManagerInference
        orig = cls.quantize_instant
        cls.quantize_instant = timed(orig)

        def cleanup():
            cls.quantize_instant = orig
            qm.__exit__()
            ctx.__exit__()
    else:
        kind = "port"
        from oracle import fq_oracle
        model, qm = pipeline.build_quantized_model(config, "cpu", quantizer_factory=fq_oracle.oracle_int_quantizer)
        qm.quantize_instant = timed(qm.quantize_instant)

        def cleanup():
            qm.detach()

    done = 0
    try:
        with torch.no_grad():
            for _ in range(warmup):
                pipeline.accuracy_counts(model(x), t)
            quant_s[0] = 0.0
            t0 = time.perf_counter()
            for _ in range(steps):
                pipeline.accuracy_counts(model(x), t)
                done += 1
                if time.perf_counter() - t0 > budget_s:
                    break
            dt = time.perf_counter() - t0
    finally:
        cleanup()
    return {"ips": batch * done / dt, "sec_per_step": dt / done, "cores": cores, "steps": done, "kind": kind,
            "quant_share": quant_s[0] / dt}


def cpu_config0(reps=50, warm=5):
    """BASELINE configs[0]: int4 per-tensor quant-dequant of one 1x64x56x56 activation on CPU through the pure-PyTorch
    int_quantizer (BASELINE.md section 3): min/max + __gemmlowpQuantize1__ (mode B) and the full Laplace call (mode D), at
    1 thread and at all host threads, median of `reps` after `warm`."""
    import torch
    from oracle import ref_live
    from oracle.host import host_threads
    p = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=False, bit_alloc_act=False,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    if ref_live.python_available():
        kind = "reference"
        ctx = ref_live.cpu_mode()
        ns = ctx.__enter__()
        make = ns.int_quantizer
    else:
        kind, ctx = "port", None
        from oracle import fq_oracle
        make = fq_oracle.oracle_int_quantizer
    torch.manual_seed(12345)
    x = torch.randn(1, 64, 56, 56)
    q_b, q_d = make("int4", dict(p)), make("int4", dict(p, clipping="laplace"))

    def med(fn):
        for _ in range(warm):
            fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        ts.sort()
        return ts[len(ts) // 2]

    out = {"kind": kind, "tensor": "1x64x56x56 fp32 (200704 elements), torch.manual_seed(12345)", "reps": reps, "warmup": warm}
    try:
        for name, threads in (("1_thread", 1), ("all_threads", host_threads())):
            torch.set_num_threads(threads)
            tb = med(lambda: q_b.__gemmlowpQuantize1__(x, x.max() - x.min(), x.min()))
            td = med(lambda: q_d(x, "conv0_activation", "activation"))
            out[name] = {"threads": threads, "minmax_quantize1_ms": tb * 1e3, "minmax_quantize1_gelem_per_s": x.numel() / tb / 1e9,
                         "laplace_call_ms": td * 1e3, "laplace_call_gelem_per_s": x.numel() / td / 1e9}
    finally:
        if ctx is not None:
            ctx.__exit__()
        torch.set_num_threads(host_threads())
    return out


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    r = cpu_pipeline(args.config, args.cpu_batch, max(1, args.steps), max(0, args.warmup), args.cpu_budget_s)
    sample = ("%d steps (of %d requested; wall-clock cap %.0f s) after %d warm-ups of %d images (of the %d-image batch) through %s, "
              "%d host threads (cgroup quota); %.0f %% of a step inside quantize_instant, the rest torch CPU convolutions" % (
                  r["steps"], args.steps, args.cpu_budget_s, args.warmup, args.cpu_batch, args.batch,
                  "the reference's own manager + IntQuantizer (oracle/_ref/pyref; compiled-leaf calls through its C restatement)"
                  if r["kind"] == "reference" else "the oracle port of int_quantizer.py", r["cores"], 100 * r["quant_share"]))
    line = {"impl": "reference", "metric": metric_name(args.config), "value": r["ips"], "unit": UNIT, "n_gpus": args.gpus,
            "steps": r["steps"], "warmup": args.warmup, "ms_per_step": r["sec_per_step"] * 1e3, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload_string(args.config, args.batch), "cpu_sample_batch": args.cpu_batch,
                       "steps_requested": args.steps},
            "cpu_baseline": {"value": r["ips"], "unit": UNIT, "cores": r["cores"], "kind": r["kind"], "sample": sample,
                             "quant_share_of_step": r["quant_share"]},
            "e2e": {"value": r["ips"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line))


# ---------------------------------------------------------------------------------------------------
# this framework
# ---------------------------------------------------------------------------------------------------
def timed_steps(torch, step, n, barrier):
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    barrier()
    return e0.elapsed_time(e1)


DUMP_BYTES = 64 << 20


def dump_outputs(directory, arrays):
    """Write each device tensor of `arrays` as `directory`/<name>.npy in float32, at most DUMP_BYTES in all: a larger
    tensor is cut to a fixed, seeded sample of its rows (same rows in every run with the same arguments)."""
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    share = DUMP_BYTES // max(len(arrays), 1)
    for name, t in sorted(arrays.items()):
        a = t.detach().float().cpu().numpy()
        if a.nbytes > share:
            rows = max(share // max(a[:1].nbytes, 1), 1)
            a = a[np.sort(np.random.RandomState(0).choice(a.shape[0], rows, replace=False))]
        np.save(os.path.join(directory, name + ".npy"), a)


def run_fqb200(args):
    import torch
    import torch.distributed as dist
    import cnn_quantization_b200 as fq
    from cnn_quantization_b200 import ops, pipeline

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (the fake-quantization path has no CPU fallback)")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    fq._lib.load()
    # cuDNN's heuristic algorithm choice, not autotuning (inference_sim.py:205 sets benchmark): autotuning picks by timing,
    # so another process may pick another convolution algorithm and the same inputs would give other outputs
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True

    model, qm = pipeline.build_quantized_model(args.config, dev, channels_last=args.channels_last)
    x_host, t_host = pipeline.synthetic_batch(args.batch, seed=1000 + rank, pin=True, channels_last=args.channels_last)
    x_dev, t_dev = x_host.to(dev), t_host.to(dev)
    total = torch.zeros(4, device=dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    last = {}

    def step_resident():
        with torch.no_grad():
            logits = model(x_dev)
            counts = pipeline.accuracy_counts(logits, t_dev)
            total.add_(counts)
        last["logits"], last["accuracy_counts"] = logits, counts

    # end to end: every step copies ITS input batch from pinned host memory and reads its 4-float metric vector back.
    # The copy of step k+1 runs on a copy stream while step k computes (double-buffered device staging), which is what
    # pipeline.validate() does for a stream of host batches.
    feeder = pipeline.HostFeeder(dev, x_host, t_host)
    host_metrics = torch.zeros(4).pin_memory()

    def step_e2e():
        with torch.no_grad():
            x, t = feeder.next()        # waits for this step's copy, starts the next step's
            host_metrics.copy_(pipeline.accuracy_counts(model(x), t), non_blocking=True)
        torch.cuda.current_stream().synchronize()  # the caller reads the step's metrics

    warm = max(args.warmup, 3)
    for _ in range(warm):
        step_resident()
    barrier()

    # ---- timed region 1: inputs resident in HBM ---------------------------------------------------
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ops.profile_reset(enable=True)
    if os.environ.get("FQB_CUDA_PROFILER"):  # ncu --profile-from-start off: capture the timed region only
        torch.cuda.profiler.start()
    ms = timed_steps(torch, step_resident, args.steps, barrier)
    if os.environ.get("FQB_CUDA_PROFILER"):
        torch.cuda.profiler.stop()
    prof = ops.profile_collect()
    ops.profile_reset(enable=False)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last)

    # ---- timed region 2: end to end from pinned host memory --------------------------------------------
    feeder.start()
    for _ in range(2):
        step_e2e()
    barrier()
    feeder.start()  # the timed region issues the copy of its first step itself
    ms_e2e = timed_steps(torch, step_e2e, args.steps, barrier)
    feeder.stop()

    # ---- BASELINE configs[3] per-GPU share (ResNet-101, 128 images per GPU) at every N ------------------
    sec = {}
    if not args.no_secondary and args.config == "resnet50_w4a4":
        sec["config3"] = secondary(args, dev, "resnet101_w4a4", 128, args.channels_last, "D", barrier)

    t_ms = torch.tensor([ms, ms_e2e, sec.get("config3", {}).get("ms_per_step", 0.0)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t_ms, op=dist.ReduceOp.MAX)
    ms, ms_e2e, ms_c3 = t_ms.tolist()
    loss, top1, top5, n_img = pipeline.reduce_metrics(total)  # the path's one collective

    if rank == 0:
        peak, peak_src = peaks()
        images = world * args.batch * args.steps
        value = images / (ms / 1e3)
        e2e = images / (ms_e2e / 1e3)
        # dominant kernel: the fused kernel in mode D (reference computation: 3 reads + 1 write = 16 B/element)
        # ... and, channels-last, the same kernel with the block's residual add + ReLU in its apply phase (mode "Dr": one
        # more read, 20 B/element).  Both are launches of ONE kernel: the headline roofline covers all of them, "parts"
        # splits it.
        dom_mode = "D" if "D" in prof["modes"] else "B"
        # (mode "S": the statistics-only launches of the shortcut convolutions of down-sampling blocks, 8 B/element; their
        # apply happens inside the "Dr" launch that consumes them)
        parts = {k: prof["modes"][k] for k in (dom_mode, dom_mode + "r", dom_mode + "p", "S") if k in prof["modes"]}
        dom = {f: sum(v[f] for v in parts.values()) for f in ("launches", "elems", "ms", "bytes")}
        achieved = (dom["bytes"] / 1e9) / (dom["ms"] / 1e3) if dom["ms"] > 0 else 0.0
        traffic, traffic_src = NCU_TRAFFIC_BYTES_PER_LAUNCH.get(
            "%s/%d/%s" % (args.config, args.batch, "nhwc" if args.channels_last else "nchw"), (None, None))
        quant_ms = sum(m["ms"] for m in prof["modes"].values())
        quant_elems = sum(m["elems"] for m in prof["modes"].values())
        kernel = "fq_cl_kernel (bulk-copy ring)" if args.channels_last else "fq_fused_kernel<4>"
        line = {
            "metric": metric_name(args.config), "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": warm,
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload_string(args.config, args.batch),
                       "parallelism": "dp%d (batch sharded per rank, one all-reduce of 4 metrics)" % world,
                       "l2": "inputs larger than L2 (308 MB input per step; hooked tensors 51 MB - 1.6 GB each, the next "
                             "layer's convolution runs between two fused launches)",
                       "memory_format": "torch.channels_last (same logical NCHW tensors and results; --nchw selects contiguous NCHW)"
                                        if args.channels_last else "contiguous NCHW",
                       "arithmetic": "fake quantization fp32; convolutions cuDNN %s with torch's default allow_tf32=True "
                                     "(third party in the reference too, same default there)" % ("NHWC" if args.channels_last else "NCHW")},
            "e2e": {"value": e2e, "unit": UNIT, "ms_per_step": ms_e2e / args.steps,
                    "h2d_bytes_per_step": x_host.numel() * 4 + t_host.numel() * 8, "d2h_bytes_per_step": 16,
                    "overlap": "H2D of step k+1 on a copy stream while step k computes (pipeline.HostFeeder)"},
            "gpu_launches": prof["launches"],
            "roofline": {"bound": "hbm", "kernel": "%s mode %s" % (kernel, " + ".join(parts) if parts else dom_mode),
                         "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak if peak else None,
                         "peak_source": peak_src, "traffic": traffic, "traffic_unit": "bytes per launch (ncu, DRAM read + write)",
                         "traffic_source": traffic_src, "launches": dom["launches"],
                         "algorithmic_bytes_per_launch": dom["bytes"] / max(dom["launches"], 1),
                         "algorithmic_bytes_per_elem": {"D": 16, "B": 12, "Dr": 20, "Br": 16, "Dp": 13, "S": "8 (mode D) / 4 (mode B)"},
                         "avg_launch_ms": dom["ms"] / max(dom["launches"], 1),
                         "parts": {k: {"launches": v["launches"], "avg_launch_ms": v["ms"] / max(v["launches"], 1),
                                       "algorithmic_bytes_per_launch": v["bytes"] / max(v["launches"], 1),
                                       "frac": (v["bytes"] / 1e9) / (v["ms"] / 1e3) / peak if v["ms"] and peak else None}
                                   for k, v in parts.items()},
                         "note": "algorithmic bytes = the reference computation's passes (SURVEY.md 8d); the channels-last "
                                 "kernel gets the std out of the first pass and small tensors stay L2-resident, so a layout "
                                 "can legitimately read above 1.0"},
            "roofline_fused_block_epilogue": (lambda r: None if not r else {
                "kernel": "%s mode D + residual add + ReLU of the block (16 of the 53 mode-D tensors of a step)" % kernel,
                "algorithmic_bytes_per_elem": 20, "launches": r["launches"], "avg_launch_ms": r["ms"] / max(r["launches"], 1),
                "achieved": (r["bytes"] / 1e9) / (r["ms"] / 1e3) if r["ms"] else None, "unit": "GB/s",
                "frac": (r["bytes"] / 1e9) / (r["ms"] / 1e3) / peak if r["ms"] else None,
                "note": "replaces a separate 12 B/element add+ReLU pass: 16 + 12 = 28 B/element become 20"})(prof["modes"].get("Dr")),
            "quant": {"gelem_per_s": quant_elems / (quant_ms / 1e3) / 1e9 if quant_ms else None,
                      "ms_per_step": quant_ms / args.steps, "share_of_step": quant_ms / ms,
                      "modes": {k: {"launches": v["launches"], "ms": v["ms"], "GBps": (v["bytes"] / 1e9) / (v["ms"] / 1e3) if v["ms"] else None}
                                for k, v in prof["modes"].items()},
                      "by_layout": {k: {"launches": v["launches"], "ms_avg": v["ms"] / v["launches"],
                                        "frac": (v["bytes"] / 1e9) / (v["ms"] / 1e3) / peak if v["ms"] else None}
                                    for k, v in sorted(prof["shapes"].items(), key=lambda kv: -kv[1]["ms"])}},
            "clocks": clocks,
            "check": {"loss": loss, "top1": top1, "top5": top5, "images": n_img},
        }
        if "config3" in sec:
            c3 = dict(sec["config3"])
            c3.update(workload=workload_string("resnet101_w4a4", 128) + " - BASELINE configs[3] (batch 1024 over 8 GPUs) at %d GPU(s)" % world,
                      ms_per_step=ms_c3, value=world * 128 / (ms_c3 / 1e3), n_gpus=world)
            line["config3_resnet101_b128"] = c3
        if world == 1 and not args.no_secondary and args.config == "resnet50_w4a4":
            line["config1_w8a8"] = secondary(args, dev, "resnet50_w8a8", args.batch, args.channels_last, "B", barrier, peak=peak)
            line["config4_vgg16"] = secondary(args, dev, "vgg16_w4a4", args.batch, args.channels_last, "D", barrier, peak=peak)
            other = not args.channels_last
            line["channels_last_variant" if other else "nchw_variant"] = secondary(
                args, dev, args.config, args.batch, other, "D", barrier, peak=peak)
            try:
                line["stats_use_variant"] = stats_use_variant(args, dev, barrier, peak)
            except Exception as e:  # a diagnostic next to the headline: never fails the run
                line["stats_use_variant"] = {"unavailable": repr(e)[:300]}
            line["kernel_bench"] = kernel_bench(torch, dev, peak)
            try:
                line["gpu_baseline"] = gpu_baseline(torch, dev, peak)
            except Exception as e:  # the checker is optional
                line["gpu_baseline"] = {"unavailable": repr(e)[:200]}
        if "config3" in sec and "roofline" in sec["config3"]:
            pass
        if world == 1 and not args.no_cpu_baseline:
            r = cpu_pipeline(args.config, args.cpu_batch, 3, 1, 120.0)
            line["cpu_baseline"] = {"value": r["ips"], "unit": UNIT, "cores": r["cores"], "kind": r["kind"],
                                    "sample": "%d steps (after 1 warm-up) of %d images through %s + torch CPU convolutions, %d host "
                                              "threads (cgroup quota); %.0f %% of a step inside quantize_instant" % (
                                                  r["steps"], args.cpu_batch,
                                                  "the reference's own manager + IntQuantizer (oracle/_ref/pyref)" if r["kind"] == "reference"
                                                  else "the oracle port of int_quantizer.py", r["cores"], 100 * r["quant_share"]),
                                    "quant_share_of_step": r["quant_share"]}
            line["config0_cpu_leaf"] = cpu_config0()
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def stats_use_variant(args, dev, barrier, peak):
    """SURVEY.md 8(f) rank 1, the reference README's best-accuracy recipe: `-sm collect` on two 32-image batches (twice,
    like the reference: per-tensor and per-channel tables, written in the reference's CSV / pickle formats; two batches
    because the reference's per-channel summary collapses the channels of a single-batch collection,
    statistic_manager_perchannel.py:163-165), then `-sm use` - every activation is an apply-only launch (mode A,
    8 B/element).  Reports the pipeline rate of the use mode."""
    import shutil
    import tempfile
    import torch
    from cnn_quantization_b200 import ops, pipeline
    base = tempfile.mkdtemp(prefix="fq_stats_")
    try:
        flags = dict(pipeline.CONFIGS[args.config], stats_folder="bench", stats_base_dir=base)
        xs, _ = pipeline.synthetic_batch(64, seed=11, channels_last=args.channels_last)
        xs = xs.to(dev)
        if args.channels_last:
            xs = xs.contiguous(memory_format=torch.channels_last)
        for pcq in (False, True):
            model, qm = pipeline.build_quantized_model(dict(flags, stats_mode="collect", per_channel_quant_act=pcq), dev,
                                                       channels_last=args.channels_last)
            with torch.no_grad():
                model(xs[:32])
                model(xs[32:])
            qm.__exit__()
            del model, qm
        model, qm = pipeline.build_quantized_model(dict(flags, stats_mode="use"), dev, channels_last=args.channels_last)
        x, t = pipeline.synthetic_batch(args.batch, seed=7, channels_last=args.channels_last)
        x, t = x.to(dev), t.to(dev)
        if args.channels_last:
            x = x.contiguous(memory_format=torch.channels_last)

        def step():
            with torch.no_grad():
                pipeline.accuracy_counts(model(x), t)

        for _ in range(3):
            step()
        ops.profile_reset(enable=True)
        ms = timed_steps(torch, step, 3, barrier) / 3
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        qm.detach()
        del model, qm, x
        torch.cuda.empty_cache()
        a = prof["modes"].get("A", {"bytes": 0, "ms": 0.0, "launches": 0})
        gbs = (a["bytes"] / 1e9) / (a["ms"] / 1e3) if a["ms"] else None
        return {"workload": workload_string(args.config, args.batch) + ", offline statistics (-sm use) collected on 2 x 32 images",
                "metric": metric_name(args.config), "value": args.batch / (ms / 1e3), "unit": UNIT, "ms_per_step": ms, "steps": 3,
                "quant_ms_per_step": sum(m["ms"] for m in prof["modes"].values()) / 3,
                "launches_per_step": {k: v["launches"] // 3 for k, v in prof["modes"].items()},
                "roofline": {"kernel": "given-parameter launches (mode A)", "algorithmic_bytes_per_elem": 8, "achieved": gbs,
                             "peak": peak, "unit": "GB/s", "frac": gbs / peak if gbs else None, "launches": a["launches"]}}
    finally:
        shutil.rmtree(base, ignore_errors=True)


def secondary(args, dev, config, batch, channels_last, mode, barrier, peak=None):
    """A short (3 timed steps, inputs resident) run of another configuration next to the headline one; reports the
    pipeline rate and the roofline of the dominant kernel mode (D: 16 B/element, B: 12 B/element)."""
    import torch
    from cnn_quantization_b200 import ops, pipeline
    if peak is None:
        peak, _ = peaks()
    model, qm = pipeline.build_quantized_model(config, dev, channels_last=channels_last)
    x, t = pipeline.synthetic_batch(batch, seed=7, channels_last=channels_last)
    x, t = x.to(dev), t.to(dev)
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)

    def step():
        with torch.no_grad():
            pipeline.accuracy_counts(model(x), t)

    for _ in range(3):
        step()
    ops.profile_reset(enable=True)
    ms = timed_steps(torch, step, 3, barrier) / 3
    prof = ops.profile_collect()
    ops.profile_reset(enable=False)
    qm.detach()
    del model, qm, x
    torch.cuda.empty_cache()
    ps = [prof["modes"][k] for k in (mode, mode + "r", mode + "p", "S") if k in prof["modes"]]
    # "r": + the block's residual add + ReLU (4 B/element more); "p": + the 2x2 max pooling behind the convolution (13 B/element:
    # the apply phase writes a quarter); "S": statistics only (8)
    b = {f: sum(v[f] for v in ps) for f in ("bytes", "ms", "launches")}
    gbs = (b["bytes"] / 1e9) / (b["ms"] / 1e3) if b["ms"] else None
    quant_ms = sum(m["ms"] for m in prof["modes"].values()) / 3
    return {"workload": workload_string(config, batch), "memory_format": "channels_last" if channels_last else "nchw",
            "metric": metric_name(config), "value": batch / (ms / 1e3), "unit": UNIT, "ms_per_step": ms, "steps": 3,
            "quant_ms_per_step": quant_ms,
            "roofline": {"kernel": "fused kernel mode %s (+ the r / p / S variants of its launches)" % mode,
                         "algorithmic_bytes_per_elem": {"D": 16, "B": 12}[mode],
                         "achieved": gbs, "peak": peak, "unit": "GB/s", "frac": gbs / peak if gbs else None,
                         "launches": b["launches"]}}


def _median_ms(torch, fn, flush, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.zero_()  # L2 flush: 256 MB written between repetitions
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def kernel_bench(torch, dev, peak):
    """The metric's first half: stand-alone quant-dequant Gelem/s and algorithmic GB/s of every kernel mode on one
    512x64x56x56 activation (411 MB), L2 flushed between repetitions, CUDA events, median of 5."""
    from cnn_quantization_b200 import _lib as L, ops
    n, c, hw = 512, 64, 56
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    x = torch.randn(n, c, hw, hw, device=dev)
    xcl = x.contiguous(memory_format=torch.channels_last)
    lay = (n, c, hw * hw)
    d = torch.rand(c, device=dev) + 1
    o = -torch.rand(c, device=dev)
    bits = torch.full((c,), 4.0, device=dev)
    out, outcl = torch.empty_like(x), torch.empty_like(xcl)
    rcl = torch.randn(n, c, hw, hw, device=dev).contiguous(memory_format=torch.channels_last)
    cases = [
        ("D_laplace_bitalloc_nhwc", 16, lambda: ops.fused(xcl, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True, out=outcl, channels_last=True)),
        ("D_laplace_bitalloc_nchw", 16, lambda: ops.fused(x, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True, out=out)),
        ("B_minmax_per_channel_nhwc", 12, lambda: ops.fused(xcl, lay, range_mode=L.RANGE_MINMAX, num_bits=4, out=outcl, channels_last=True)),
        ("B_minmax_per_sample_int8", 12, lambda: ops.fused(x, (1, n, c * hw * hw), scope=L.SCOPE_GROUP_MEAN, leaf=L.LEAF_COMPILED, num_bits=8, out=out)),
        ("A_given_per_channel_nhwc", 8, lambda: ops.quantize1(xcl, d, o, 4, bits=bits, layout=lay, out=outcl)),
        ("A_given_per_channel_nchw", 8, lambda: ops.quantize1(x, d, o, 4, bits=bits, layout=lay, out=out)),
        ("A_given_per_tensor", 8, lambda: ops.quantize1(x, d[:1], o[:1], 4, out=out)),
        ("a1_float2gemmlowp", 8, lambda: ops.float2gemmlowp(x, 7.0, -3.0, 8, False, True, None, out=out)),
        # the launches that also finish what surrounds the convolution (bytes = what THIS launch has to move)
        ("Dr_laplace_bitalloc_block_epilogue_nhwc", 20, lambda: ops.fused(xcl, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True,
                                                                            out=outcl, channels_last=True, residual=rcl, residual_relu=True)),
        ("S_statistics_only_nhwc", 8, lambda: ops.fused(xcl, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True,
                                                          channels_last=True, stats_only=True)),
        ("Dp_laplace_bitalloc_pool2x2_nhwc", 13, lambda: ops.fused(xcl, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True,
                                                                     channels_last=True, positive=True, pool=(2, 2))),
        ("Ar_given_block_epilogue_nhwc", 12, lambda: ops.fused(xcl, lay, range_mode=L.RANGE_GIVEN, num_bits=4, given=(d, o, bits),
                                                                 out=outcl, channels_last=True, residual=rcl, residual_relu=True)),
        ("torch_copy_reference_point", 8, lambda: out.copy_(x)),
    ]
    res = {"tensor": "512x64x56x56 fp32 (411 MB)", "l2": "flushed between repetitions (256 MB memset)", "reps": 5}
    for name, bpe, fn in cases:
        ms = _median_ms(torch, fn, flush)
        gbs = x.numel() * bpe / ms / 1e6
        res[name] = {"ms": ms, "gelem_per_s": x.numel() / ms / 1e6, "algorithmic_bytes_per_elem": bpe, "GBps": gbs, "frac": gbs / peak}
    return res


def gpu_baseline(torch, dev, peak):
    """The 'kernel to beat' (BASELINE.md section 3, SURVEY 8c/8d): the reference's own code on the same GPU and tensor
    (512x64x56x56) - its compiled extension incl. the zeros_like / noise tensor of its wrapper, and its pure-PyTorch
    per-channel W4A4 path - next to ours.  Checker code (oracle/_ref) is timed here, never used by the product path."""
    import cnn_quantization_b200 as fq
    from oracle import ref_live
    if not ref_live.available():
        return {"unavailable": "oracle/_ref not built"}
    ns = ref_live.load()
    ext = ref_live.load_extension()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    n, c, hw = 512, 64, 56
    x = torch.randn(n, c, hw, hw, device=dev)
    xcl = x.contiguous(memory_format=torch.channels_last)
    p = dict(clipping="laplace", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=True,
             bit_alloc_weight=True, bcorr_act=False, bcorr_weight=True, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    p8 = dict(p, clipping="no", pcq_act=False)
    rq4, rq8 = ns.int_quantizer("int4", dict(p)), ns.int_quantizer("int8", dict(p8))
    q4, q8 = fq.int_quantizer("int4", dict(p)), fq.int_quantizer("int8", dict(p8))
    el = x.numel()

    def row(ms, bpe):
        return {"ms": ms, "gelem_per_s": el / ms / 1e6, "GBps_algorithmic": el * bpe / ms / 1e6, "frac": el * bpe / ms / 1e6 / peak}

    res = {"tensor": "512x64x56x56 fp32 (411 MB)", "l2": "flushed between repetitions", "reps": 3}
    t = _median_ms(torch, lambda: rq4(x, "conv1_activation", "activation"), flush, 3)
    res["reference_per_channel_w4a4_pytorch_on_gpu"] = row(t, 16)
    t2 = _median_ms(torch, lambda: q4(xcl, "conv1_activation", "activation"), flush, 3)
    res["ours_per_channel_w4a4_nhwc"] = row(t2, 16)
    t3 = _median_ms(torch, lambda: q4(x, "conv1_activation", "activation"), flush, 3)
    res["ours_per_channel_w4a4_nchw"] = row(t3, 16)
    res["speedup_per_channel_w4a4"] = t / min(t2, t3)
    t = _median_ms(torch, lambda: rq8(x, "maxpool0_out", "activation_pooling"), flush, 3)
    res["reference_int8_minmax_compiled_kernel_path"] = row(t, 12)
    t2 = _median_ms(torch, lambda: q8(x, "maxpool0_out", "activation_pooling"), flush, 3)
    res["ours_int8_minmax_fused"] = row(t2, 12)
    res["speedup_int8_minmax"] = t / t2
    t = _median_ms(torch, lambda: ext.float2gemmlowp(x, 7.0, -3.0, 8, False, True, torch.zeros_like(x)), flush, 3)
    res["reference_float2gemmlowp_with_its_noise_tensor"] = row(t, 8)
    out = torch.empty_like(x)
    t2 = _median_ms(torch, lambda: fq.ops.float2gemmlowp(x, 7.0, -3.0, 8, False, True, None, out=out), flush, 3)
    res["ours_float2gemmlowp"] = row(t2, 8)
    res["speedup_float2gemmlowp"] = t / t2
    return res


def main():
    args = parse()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_fqb200(args)


if __name__ == "__main__":
    main()
