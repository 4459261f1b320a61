"""HBM traffic of the set-abstraction shared MLP (3 -> 64 -> 128 -> 256, BatchNorm train mode, ReLU, max over 64
neighbours) forward + backward at the BASELINE size (8 scenes x 2048 seeds x 64 neighbours = 1 048 576 rows).

    ncu --profile-from-start off --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum \
        --csv --log-file out.csv python tools/sa_mlp_traffic.py
    python tools/sa_mlp_traffic.py --summarise out.csv      -> total bytes / time per direction

Works with any revision of the package on PYTHONPATH, so two revisions can be compared the same way."""
import csv
import sys
from pathlib import Path


def summarise(path):
    rows = []
    with open(path) as f:
        lines = [l for l in f if l.startswith('"')]
    rd = csv.DictReader(lines)
    per = {}
    for r in rd:
        per.setdefault((r["ID"], r["Kernel Name"]), {})[r["Metric Name"]] = (float(r["Metric Value"].replace(",", "")), r["Metric Unit"])
    unit = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-9, "us": 1e-6, "ms": 1e-3, "usecond": 1e-6,
            "nsecond": 1e-9, "msecond": 1e-3, "second": 1.0}
    tot_r = tot_w = tot_t = 0.0
    print(f"{'read MB':>10} {'write MB':>10} {'us':>9}  kernel")
    for (kid, name), m in per.items():
        r = m["dram__bytes_read.sum"][0] * unit[m["dram__bytes_read.sum"][1]]
        w = m["dram__bytes_write.sum"][0] * unit[m["dram__bytes_write.sum"][1]]
        t = m["gpu__time_duration.sum"][0] * unit[m["gpu__time_duration.sum"][1]]
        tot_r, tot_w, tot_t = tot_r + r, tot_w + w, tot_t + t
        print(f"{r / 1e6:10.1f} {w / 1e6:10.1f} {t * 1e6:9.1f}  {name[:90]}")
    print(f"TOTAL dram read {tot_r / 1e9:.3f} GB + write {tot_w / 1e9:.3f} GB = {(tot_r + tot_w) / 1e9:.3f} GB over "
          f"{len(per)} launches, {tot_t * 1e3:.3f} ms summed (cold-cache, serialised)")


def main():
    import torch

    sys.path.insert(0, str(Path(__file__).resolve().parents[1])) if "--r1" not in sys.argv else None
    from coda_neurips2023_b200.pointnet2.pytorch_utils import SharedMLP

    torch.manual_seed(0)
    b, p, s = 8, 2048, 64
    mlp = SharedMLP([3, 64, 128, 256], bn=True).cuda().train()
    x = (torch.rand(b, 3, p, s, device="cuda") - 0.5)
    g = torch.randn(b, 256, p, device="cuda")

    def step():
        for q in mlp.parameters():
            q.grad = None
        y = mlp.forward_max_pooled(x)
        assert y is not None, "fused SA path not taken"
        y.backward(g)
        return y

    step()
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    step()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        step()
    e1.record()
    torch.cuda.synchronize()
    print(f"SA shared MLP fwd+bwd: {e0.elapsed_time(e1) / 5:.3f} ms per iteration (CUDA events, warm)")


if __name__ == "__main__":
    if "--summarise" in sys.argv:
        summarise(sys.argv[sys.argv.index("--summarise") + 1])
    else:
        main()
