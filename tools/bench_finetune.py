"""Step time of fine-tuning modes on the native trainer, at tools/bench_train.py's workload (batch 64 @352x352, train-mode forward
-> device loss -> backward -> flat-bucket SGD step).  Four modes on one model, alternated round by round so that clock and neighbour
noise falls on all of them alike:

    all        every parameter trainable, every BatchNorm layer in train mode (train.py)
    bb         the backbone frozen (requires_grad=False); its BatchNorm layers still use batch statistics
    bb+evalbn  the backbone frozen and its BatchNorm layers in .eval() (train_dist.py --freeze backbone --freeze-bn)
    heads      only the FPN and heads trainable (the backbone and the 1x1 reductions conv1x1_2 / conv1x1_3 frozen)

Each mode keeps its own FlatGradBucket and SGD optimizer over the trainable parameters.  Prints one JSON line per mode (median and
spread of the per-round step times, CUDA events around each round) with the card's name and power limit.
    python tools/bench_finetune.py [rounds] [steps per round]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import yfv2  # noqa: E402,F401
import synth  # noqa: E402
import model.detector as det  # noqa: E402
import utils.loss as ul  # noqa: E402
import train_ddp  # noqa: E402

MODES = {
    "all": ((), False),
    "bb": (("backbone.",), False),
    "bb+evalbn": (("backbone.",), True),
    "heads": (("backbone.", "fpn.conv1x1_"), False),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def set_mode(m, frozen, eval_bn):
    m.train()
    for n, p in m.named_parameters():
        p.requires_grad_(not n.startswith(frozen) if frozen else True)
    if eval_bn:
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d) and not mod.weight.requires_grad and not mod.bias.requires_grad:
                mod.eval()


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune.py: needs a CUDA device")
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    N = 64
    torch.manual_seed(2)
    m = det.Detector(80, 3, True).cuda().train()
    x = torch.rand(N, 3, 352, 352).cuda()
    targets = synth.make_targets(2, N).cuda()
    cfg = synth.coco_cfg()
    state = {}
    for name, (frozen, eval_bn) in MODES.items():
        set_mode(m, frozen, eval_bn)
        for p in m.parameters():
            p.grad = None
        bucket = train_ddp.FlatGradBucket(m.parameters())
        opt = torch.optim.SGD([p for p in m.parameters() if p.requires_grad], lr=1e-6, momentum=0.949, weight_decay=0.0005)
        state[name] = (bucket, opt, sum(p.numel() for p in m.parameters() if p.requires_grad))
    times = {k: [] for k in MODES}
    ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(rounds + 1):                           # round 0 warms every mode up (graph captures, allocator)
        for name, (frozen, eval_bn) in MODES.items():
            bucket, opt, _ = state[name]
            set_mode(m, frozen, eval_bn)
            for p in m.parameters():
                p.grad = None
            bucket.reattach()
            train_ddp.train_step(m, bucket, opt, x, targets, cfg, ul.compute_loss)
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(steps):
                train_ddp.train_step(m, bucket, opt, x, targets, cfg, ul.compute_loss)
            ev[1].record()
            ev[1].synchronize()
            if r > 0:
                times[name].append(ev[0].elapsed_time(ev[1]) / steps)
    gpu = gpu_info()
    base = float(np.median(times["all"]))
    for name in MODES:
        t = np.array(times[name])
        print(json.dumps({"mode": name, "trainable_floats": state[name][2], "batch": N, "size": 352, "ms_per_step": round(float(np.median(t)), 3),
                          "min": round(float(t.min()), 3), "max": round(float(t.max()), 3), "vs_all": round(float(np.median(t)) / base, 3),
                          "rounds": rounds, "steps_per_round": steps, "gpu": gpu}))


if __name__ == "__main__":
    main()
