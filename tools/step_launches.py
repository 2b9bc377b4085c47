"""One training step's launch list out of an `ncu --metrics gpu__time_duration.sum --csv` log of bench.py: finds the
period of the kernel-name sequence at the end of the log (graph replays repeat the step) and aggregates ONE period.

    python tools/step_launches.py launches.csv [top]
"""
import collections
import csv
import sys


def main(path, top=60):
    lines = [l for l in open(path, errors="replace") if not l.startswith("==")]
    seq = []
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(row["Metric Value"].replace(",", ""))
        unit = row["Metric Unit"]
        v = v / 1e3 if unit == "ns" else v * 1e3 if unit == "ms" else v * 1e6 if unit in ("s", "second") else v
        seq.append((row["Kernel Name"], v))
    names = [s[0] for s in seq]
    n = len(names)
    period = None
    for p in range(20, n // 2 + 1):
        if names[n - p:] == names[n - 2 * p:n - p]:
            period = p
            break
    if period is None:
        print(f"no repeating period found in {n} launches; aggregating everything")
        period = n
    step = seq[n - period:]
    agg = collections.defaultdict(lambda: [0, 0.0])
    for k, v in step:
        agg[k][0] += 1
        agg[k][1] += v
    tot = sum(v[1] for v in agg.values())
    ours = sum(v[0] for k, v in agg.items() if "b200gan" in k)
    ours_us = sum(v[1] for k, v in agg.items() if "b200gan" in k)
    print(f"one step = {period} launches, {tot:.1f} us serialised under ncu (cold caches); libb200gan kernels: {ours} launches, "
          f"{ours_us:.1f} us ({100 * ours_us / tot:.1f}%); other (torch/cuBLAS/NCCL): {period - ours} launches, {tot - ours_us:.1f} us")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])[:top]:
        print(f"{v[1]:10.1f} us {100 * v[1] / tot:5.1f}%  n={v[0]:4d}  avg {v[1] / v[0]:8.1f} us  {k[:150]}")


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 60)
