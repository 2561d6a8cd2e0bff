"""What the GPU bench scripts in this directory share: the repository on sys.path, the card a result was taken on, CUDA-event
timing, the median they report, the build they measure and the JSON file they write."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    """'name, power limit' of the first GPU as nvidia-smi reports them, or 'unknown'."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def timed(fn, reps=1):
    """CUDA-event times in ms of ``reps`` calls of ``fn``, each followed by a device synchronisation."""
    import torch
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def median(v):
    return sorted(v)[len(v) // 2]


def build_or_exit(tool):
    """Exit unless there is a CUDA device, then build the library the tool measures."""
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("%s measures on a CUDA device; none found" % tool)
    import __graft_entry__
    __graft_entry__.build()


def write_json(res, path):
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        json.dump(res, f)
        f.write("\n")
