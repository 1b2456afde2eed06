"""Turns ncu CSV logs into per-launch summaries.  Test/measurement infrastructure.

  launches  <ncu --metrics gpu__time_duration.sum --csv log>            -> per-kernel time shares of the whole command
  step      <ncu --metrics dram__bytes_read.sum,... --csv log> <names>  -> per-step DRAM bytes / tensor-pipe % (JSON + table)
  full      <ncu -i rep --page raw --csv export> <names>                -> per-launch table of the --set full capture
  table     <ncu --metrics ... --csv log>                               -> per-launch table without layer names

<names> is a bench.py --profile-out file: its launch order is the order of the conv launches of one step.
"""
import csv
import json
import sys
from collections import OrderedDict, defaultdict


def _rows(path):
    with open(path, newline="") as f:
        lines = [ln for ln in f if ln.startswith('"')]
    return list(csv.DictReader(lines))


def _names(path):
    out = []
    for ln in open(path):
        if ln.startswith("#") or not ln.strip():
            continue
        out.append(ln[:36].strip())
    return out


def launches(path):
    rows = _rows(path)
    t = defaultdict(float)
    n = defaultdict(int)
    for r in rows:
        if r["Metric Name"] != "gpu__time_duration.sum":
            continue
        v = float(r["Metric Value"].replace(",", ""))
        if r["Metric Unit"] in ("nsecond", "ns"):
            v /= 1e3
        elif r["Metric Unit"] in ("msecond", "ms"):
            v *= 1e3
        t[r["Kernel Name"]] += v
        n[r["Kernel Name"]] += 1
    tot = sum(t.values())
    print(f"# cold-cache serialised per-launch times: compare SHARES, not absolutes. {sum(n.values())} launches captured.")
    for k in sorted(t, key=lambda k: -t[k]):
        print(f"{t[k]:12.1f} us {100 * t[k] / tot:6.2f}%  {n[k]:3d} launches  {k}")


def _by_id(rows):
    d = OrderedDict()
    for r in rows:
        e = d.setdefault(r["ID"], {"Kernel Name": r["Kernel Name"], "Block Size": r["Block Size"]})
        v = r["Metric Value"].replace(",", "")
        try:
            v = float(v)
        except ValueError:
            pass
        e[r["Metric Name"]] = (v, r["Metric Unit"])
    return list(d.values())


def _scale(v, unit, want):
    f = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "nsecond": 1e-3, "ns": 1e-3, "usecond": 1, "us": 1, "msecond": 1e3, "ms": 1e3}
    if want == "byte":
        return v * f[unit]
    if want == "us":
        return v * f[unit]
    return v


def step(path, names_path, command=""):
    ls = _by_id(_rows(path))
    names = _names(names_path)
    rd = wr = t = tw = 0.0
    print("# layer | kernel | time us | tensor pipe % | dram read MB | dram write MB")
    for i, e in enumerate(ls):
        r = _scale(*e["dram__bytes_read.sum"], "byte")
        w = _scale(*e["dram__bytes_write.sum"], "byte")
        us = _scale(*e["gpu__time_duration.sum"], "us")
        tp = e["sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"][0]
        rd += r; wr += w; t += us; tw += us * tp
        nm = names[i] if i < len(names) else "?"
        print(f"{nm} | {e['Kernel Name']} | {us:.1f} | {tp:.1f} | {r / 1e6:.1f} | {w / 1e6:.1f}")
    js = {"command": command, "workload": "B=128,T=5 (640 crops), one step", "dram_read_bytes": rd, "dram_write_bytes": wr,
          "launches": len(ls), "serialized_time_ms": t / 1e3, "time_weighted_tensor_pipe_active_pct": tw / t if t else None}
    print("# JSON " + json.dumps(js))


def table(path):
    """Per-launch table of an ncu --metrics CSV log (no layer names): kernel, time, tensor pipe %, DRAM MB, achieved GB/s."""
    ls = _by_id(_rows(path))
    print("# kernel | time us | tensor pipe % | dram read MB | dram write MB | DRAM GB/s | dram throughput % of peak")
    for e in ls:
        r = _scale(*e["dram__bytes_read.sum"], "byte")
        w = _scale(*e["dram__bytes_write.sum"], "byte")
        us = _scale(*e["gpu__time_duration.sum"], "us")
        tp = e["sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"][0]
        dt = e.get("dram__throughput.avg.pct_of_peak_sustained_elapsed", (float("nan"), ""))[0]
        print(f"{e['Kernel Name']} | {us:.1f} | {tp:.1f} | {r / 1e6:.2f} | {w / 1e6:.2f} | {(r + w) / us / 1e3:.0f} | {dt:.1f}")


FULL_COLS = ["gpu__time_duration.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
             "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
             "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
             "l1tex__throughput.avg.pct_of_peak_sustained_active", "l1tex__m_xbar2l1tex_read_bytes.sum",
             "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "launch__registers_per_thread"]


def full(path, names_path):
    """`ncu -i rep --page raw --csv`: one row per launch, one column per metric, a units row first."""
    with open(path, newline="") as f:
        lines = [ln for ln in f if ln.startswith('"')]
    rd = list(csv.reader(lines))
    hdr, units, rows = rd[0], rd[1], rd[2:]
    names = _names(names_path)
    idx = {h: i for i, h in enumerate(hdr)}
    cols = [c for c in FULL_COLS if c in idx]
    print("# layer | Kernel Name | Block Size | " + " | ".join(f"{c} [{units[idx[c]]}]" for c in cols))
    for i, r in enumerate(rows):
        nm = names[i] if i < len(names) else "?"
        print(" | ".join([nm, r[idx["Kernel Name"]], r[idx["Block Size"]]] + [r[idx[c]] for c in cols]))


if __name__ == "__main__":
    cmd = sys.argv[1]
    if cmd == "launches":
        launches(sys.argv[2])
    elif cmd == "step":
        step(sys.argv[2], sys.argv[3], sys.argv[4] if len(sys.argv) > 4 else "")
    elif cmd == "table":
        table(sys.argv[2])
    elif cmd == "full":
        full(sys.argv[2], sys.argv[3])
    else:
        raise SystemExit(__doc__)
