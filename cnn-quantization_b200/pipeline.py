"""Inference pipeline around the fake-quantization hot path: the part of the reference's
``inference/inference_sim.py`` (``InferenceModel.__init__`` :131-229, ``validate`` :278-343) that the benchmark
needs, on synthetic ImageNet-shaped batches and random-init torchvision weights (no dataset / checkpoints offline).

One process per GPU: each rank builds the same seeded model, quantizes the same weights (deterministic, so no
broadcast), runs its shard of the batch, and the four validation counters are combined with ONE all-reduce at the
end (the reference uses single-process ``torch.nn.DataParallel``, inference_sim.py:196-200).  On-the-fly statistics
are therefore per shard - exactly what DataParallel replicas compute in the reference (SURVEY.md 8e).
"""
import torch
import torch.nn as nn

from . import manager as M

__all__ = ["CONFIGS", "INPUT_SIZE", "ARCH_KWARGS", "PAPER_NETS", "PAPER_TABLE", "paper_cell_input_size", "build_paper_cell",
           "build_quantized_model", "synthetic_batch", "validate", "accuracy_counts", "reduce_metrics", "HostFeeder"]

# BASELINE.json configs -> reference CLI flags
_W4A4 = dict(qtype="int4", qweight="int4", clipping="laplace", per_channel_quant_weights=True, per_channel_quant_act=True,
             bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True)
CONFIGS = {
    "resnet50_w8a8": dict(arch="resnet50", qtype="int8", qweight="int8"),
    "resnet50_w4a4": dict(arch="resnet50", **_W4A4),
    "resnet101_w4a4": dict(arch="resnet101", **_W4A4),
    "vgg16_w4a4": dict(arch="vgg16", bit_alloc_target_act=5.3, bit_alloc_target_weight=5.3, **_W4A4),
    "vgg16_w4a4_mtq": dict(arch="vgg16", bit_alloc_target_act=5.3, bit_alloc_target_weight=5.3, mid_thread_quant=True, **_W4A4),
    "resnet18_w4a4": dict(arch="resnet18", **_W4A4),
    # the paper's two remaining networks, "all methods combined" at 4W4A
    "inception_v3_w4a4": dict(arch="inception_v3", **_W4A4),
    "vgg16_bn_w4a4": dict(arch="vgg16_bn", **_W4A4),
}
# the square crop the reference's validation transform takes (inference_sim.py:217-218)
INPUT_SIZE = {name: 299 if cfg["arch"] == "inception_v3" else 224 for name, cfg in CONFIGS.items()}
# constructor keywords of the torchvision model, as ``pretrained=True`` builds it in the reference (the checkpoint itself is
# not loaded).  Inception-v3's auxiliary head only runs in training, but its two convolutions and its linear take ids in
# construction order and its weights are quantized, which the reference's max_mse_order_id (conv0..conv95) presumes.
ARCH_KWARGS = {"inception_v3": dict(aux_logits=True, transform_input=True, init_weights=False)}

# The paper's results table (the reference's fig/experiments.png): six networks, three bit-width settings with their method
# rows, and an FP32 column.  The paper gives no command lines; the cells read its section headings literally, with the
# shared flags of the reference README's two commands:
#
#   setting  common flags                                              method -> added flags
#   8W4A     qtype=int4, qweight=int8, per_channel_quant_act           baseline: none; aciq: clipping=laplace;
#                                                                      bit_alloc: bit_alloc_act;
#                                                                      aciq_bit_alloc: clipping=laplace, bit_alloc_act
#   4W8A     qtype=int8, qweight=int4, per_channel_quant_weights       baseline: none; bias_corr: bias_corr_weight;
#                                                                      bit_alloc: bit_alloc_weight;
#                                                                      bias_corr_bit_alloc: bit_alloc_weight, bias_corr_weight
#   4W4A     qtype=int4, qweight=int4, per_channel_quant_weights,      baseline: none; all: clipping=laplace, bit_alloc_act,
#            per_channel_quant_act                                     bit_alloc_weight, bias_corr_weight
#   FP32     q_off=True                                                fp32: one cell per network
#
# 6 x (4 + 4 + 2 + 1) = 66 cells, keyed (net, setting, method) with the torchvision arch name as net; each value is the
# ``make_args`` keywords of the cell, arch included.  Every cell uses the default bit-allocation target (the bit width).
# So the "4W4A all" cell equals ``CONFIGS["<net>_w4a4"]`` for resnet18/50/101, inception_v3 and vgg16_bn, but not for
# vgg16: ``vgg16_w4a4`` is BASELINE's bin-allocation run at a 5.3-bit target, not the paper's cell.
PAPER_NETS = ("vgg16", "vgg16_bn", "inception_v3", "resnet18", "resnet50", "resnet101")
_PAPER_SETTINGS = {
    "8W4A": (dict(qtype="int4", qweight="int8", per_channel_quant_act=True), {
        "baseline": {}, "aciq": dict(clipping="laplace"), "bit_alloc": dict(bit_alloc_act=True),
        "aciq_bit_alloc": dict(clipping="laplace", bit_alloc_act=True)}),
    "4W8A": (dict(qtype="int8", qweight="int4", per_channel_quant_weights=True), {
        "baseline": {}, "bias_corr": dict(bias_corr_weight=True), "bit_alloc": dict(bit_alloc_weight=True),
        "bias_corr_bit_alloc": dict(bit_alloc_weight=True, bias_corr_weight=True)}),
    "4W4A": (dict(qtype="int4", qweight="int4", per_channel_quant_weights=True, per_channel_quant_act=True), {
        "baseline": {}, "all": dict(clipping="laplace", bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True)}),
    "FP32": (dict(q_off=True), {"fp32": {}}),
}
PAPER_TABLE = {(net, setting, method): dict(arch=net, **common, **added)
               for net in PAPER_NETS for setting, (common, methods) in _PAPER_SETTINGS.items()
               for method, added in methods.items()}


def paper_cell_input_size(cell):
    """The square crop of a PAPER_TABLE cell, ``(net, setting, method)``: 299 for Inception-v3, 224 otherwise."""
    return 299 if cell[0] == "inception_v3" else 224


def build_paper_cell(cell, device, seed=12345, quantizer_factory=None, channels_last=False):
    """``build_quantized_model`` for a PAPER_TABLE cell, ``(net, setting, method)``: (model, manager)."""
    return build_quantized_model(PAPER_TABLE[tuple(cell)], device, seed=seed, quantizer_factory=quantizer_factory,
                                 channels_last=channels_last)


def build_quantized_model(config, device, seed=12345, quantizer_factory=None, channels_last=False):
    """Model creation as in InferenceModel.__init__: seeded random-init torchvision model (the reference loads
    pretrained weights; none are available offline), node names, before-relu marks and BN folding for ResNets,
    ``.to(device)``, ``quantize_model``.  Returns (model, manager); the manager stays attached and enabled."""
    import torchvision.models as models
    flags = dict(CONFIGS[config]) if isinstance(config, str) else dict(config)
    args = M.make_args(**flags)
    qm = M.QuantizationManagerInference(args, M.get_params(args), quantizer_factory=quantizer_factory)
    qm.enable()
    try:
        torch.manual_seed(seed)  # inference_sim.py:127
        model = models.__dict__[args.arch](weights=None, **ARCH_KWARGS.get(args.arch, {}))
    finally:
        qm.stop_stamping()
    M.set_node_names(model)
    if "resnet" in args.arch:
        M.resnet_mark_before_relu(model)
    if "resnet" in args.arch or args.arch in ("vgg16_bn", "inception_v3"):
        M.search_absorbe_bn(model)
        qm.bn_folding = True
    model.eval()
    model.to(device)
    if channels_last:
        model.to(memory_format=torch.channels_last)
    if qm.quantize:   # without a qtype (the FP32 column: q_off alone) there are no weight quantizers; the weights stay fp32
        qm.quantize_model(model)
    qm.attach(model)
    return model, qm


def synthetic_batch(batch, seed, device="cpu", hw=None, pin=False, channels_last=False, config=None):
    """ImageNet-shaped input batch + labels; N(0,1) per pixel is what a normalised image roughly looks like.  ``hw``
    defaults to the crop of ``config`` (``INPUT_SIZE``), 224 without one."""
    if hw is None:
        hw = INPUT_SIZE.get(config, 224)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, 3, hw, hw, generator=g)
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 1000, (batch,), generator=g)
    if pin and torch.cuda.is_available():
        x, t = x.pin_memory(), t.pin_memory()
    if device != "cpu":
        x, t = x.to(device, non_blocking=True), t.to(device, non_blocking=True)
    return x, t


def accuracy_counts(output, target):
    """[loss_sum, correct@1, correct@5, count] as a device tensor (no host sync): the sums behind the reference's
    AverageMeters (inference_sim.py:319-325, utils/meters.py:81-95)."""
    loss_sum = nn.functional.cross_entropy(output, target, reduction="sum")
    _, pred = output.topk(5, 1, True, True)
    hit = pred.eq(target.view(-1, 1))
    c1 = hit[:, :1].sum()
    c5 = hit.sum()
    return torch.stack([loss_sum.float(), c1.float(), c5.float(), torch.tensor(float(target.numel()), device=output.device)])


class HostFeeder(object):
    """Double-buffered host -> device staging on a copy stream: while the model runs on batch k (current stream), batch
    k+1 is copied from (pinned) host memory into the other device buffer.  The reference's ``validate`` copies every
    batch in front of its forward (inference_sim.py:300-303); with 308 MB per 512-image batch that serialised copy was
    13 % of a step.

        feeder = HostFeeder(device, x_host, t_host)      # one fixed batch, re-fed every step (bench.py), or
        feeder = HostFeeder(device); feeder.start(iter)  # an iterator of (x_host, t_host) batches (validate)
    """

    def __init__(self, device, x_host=None, t_host=None):
        self.dev = torch.device(device)
        self.copy_stream = torch.cuda.Stream(self.dev)
        self.fixed = (x_host, t_host) if x_host is not None else None
        self.src = None
        self.bufs = [None, None]
        self.ready = [None, None]
        self.pending = None   # slot whose copy has been issued and not consumed yet
        self.k = 0

    def _issue(self, slot, x_host, t_host):
        bx = self.bufs[slot]
        if bx is None or bx[0].shape != x_host.shape or bx[0].stride() != x_host.stride() or bx[1].shape != t_host.shape:
            bx = self.bufs[slot] = (torch.empty_like(x_host, device=self.dev), torch.empty_like(t_host, device=self.dev))
        # everything that read this buffer (two steps ago) has been enqueued on the current stream before this point
        free = torch.cuda.Event()
        free.record(torch.cuda.current_stream(self.dev))
        self.copy_stream.wait_event(free)
        with torch.cuda.stream(self.copy_stream):
            bx[0].copy_(x_host, non_blocking=True)
            bx[1].copy_(t_host, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.ready[slot] = ev
        self.pending = slot

    def _fetch(self):
        if self.fixed is not None:
            return self.fixed
        try:
            return next(self.src)
        except StopIteration:
            return None

    def start(self, batches=None):
        """Issue the copy of the first batch (inside the caller's timed region, if any)."""
        if batches is not None:
            self.src = iter(batches)
        self.pending = None
        first = self._fetch()
        if first is not None:
            self._issue(self.k & 1, *first)

    def next(self):
        """(x, t) of the current batch on the device - the current stream waits for its copy - or None at the end; the
        copy of the following batch starts before this returns."""
        if self.pending is None:
            return None
        slot = self.pending
        torch.cuda.current_stream(self.dev).wait_event(self.ready[slot])
        cur = self.bufs[slot]
        self.k += 1
        self.pending = None
        nxt = self._fetch()
        if nxt is not None:
            self._issue(self.k & 1, *nxt)
        return cur

    def stop(self):
        self.copy_stream.synchronize()
        self.pending = None


def validate(model, batches, device):
    """``validate()`` of the reference on an iterable of (input, target) host batches: H2D copy (double-buffered on a copy
    stream when the model lives on a GPU), forward through the hooked model, metric accumulation on the device.  Returns
    the 4-vector of accuracy_counts summed over batches."""
    total = torch.zeros(4, device=device)
    with torch.no_grad():
        if torch.device(device).type != "cuda":
            for x, t in batches:
                total += accuracy_counts(model(x.to(device)), t.to(device))
            return total
        feeder = HostFeeder(device)
        feeder.start(batches)
        while True:
            cur = feeder.next()
            if cur is None:
                break
            total += accuracy_counts(model(cur[0]), cur[1])
        feeder.stop()
    return total


def reduce_metrics(total):
    """The only collective of the path: all-reduce(SUM) of [loss_sum, correct@1, correct@5, count] over the ranks,
    then (loss, top1 %, top5 %) like the reference's AverageMeter averages."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(total, op=dist.ReduceOp.SUM)
    loss_sum, c1, c5, n = total.tolist()
    return loss_sum / n, 100.0 * c1 / n, 100.0 * c5 / n, int(n)
