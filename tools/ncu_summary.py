"""Summarise ncu captures into small text files.
  python tools/ncu_summary.py launches <csv>            -> per-kernel totals and shares
  python tools/ncu_summary.py kernel <file.ncu-rep>     -> key metrics + top stall reasons + hottest SASS lines
"""
import collections
import csv
import io
import re
import subprocess
import sys


def short_name(sig: str) -> str:
    """'void panel::panel_update_kernel<lbg::Cfg<64, 2, 16, 0>, (bool)0>(const double *, ...)' -> 'panel_update_kernel<Cfg<64,2,16,0>,0>'"""
    sig = sig.replace("(bool)", "").replace("(anonymous namespace)::", "").replace("<unnamed>::", "")
    depth, cut = 0, len(sig)
    for i, ch in enumerate(sig):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            cut = i
            break
    sig = sig[:cut]
    m = re.match(r"([^<]*)(<.*>)?", sig)
    base = (m.group(1).split("::")[-1].split() or ["?"])[-1]
    return base + (m.group(2) or "").replace("lbg::", "").replace(" ", "")


def launches(path):
    rows = [r for r in csv.reader(open(path)) if len(r) > 10]
    hdr = rows[0]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = collections.defaultdict(lambda: [0, 0.0])
    for r in rows[1:]:
        name = short_name(r[ki])
        v = float(r[vi].replace(",", ""))
        v *= {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(r[ui], 1e-6)
        agg[name][0] += 1
        agg[name][1] += v
    tot = sum(v[1] for v in agg.values())
    print(f"# ncu --metrics gpu__time_duration.sum --clock-control none  ({path}); cold-cache, serialised: compare shares")
    for k, v in sorted(agg.items(), key=lambda x: -x[1][1]):
        print(f"{k:52s} launches={v[0]:5d} total_ms={v[1]:10.3f} share={v[1] / tot:6.3f}")
    print(f"{'TOTAL':52s} launches={sum(v[0] for v in agg.values()):5d} total_ms={tot:10.3f}")


WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_tensor_subpipe_dmma.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active_realtime",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "sm__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "lts__t_sector_hit_rate.pct", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__cycles_elapsed.avg.per_second", "launch__shared_mem_per_block_dynamic", "smsp__inst_executed.sum"]


def kernel(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    h, u, v = rows[0], rows[1], rows[-1]
    print(f"# {path}: {v[h.index('Kernel Name')] if 'Kernel Name' in h else ''}")
    stalls = []
    for i, n in enumerate(h):
        if any(n == w or n.endswith(w) or (w in n and "realtime" in w) for w in WANT):
            print(f"{n:90s} {v[i]:>16s} {u[i]}")
        if "smsp__average_warps_issue_stalled" in n and n.endswith("per_issue_active.ratio"):
            try:
                stalls.append((float(v[i]), n.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", "")))
            except ValueError:
                pass
    print("# warp stall reasons (warps per issue-active cycle), top 6")
    for s, n in sorted(stalls, reverse=True)[:6]:
        print(f"  {n:28s} {s:8.3f}")
    src = subprocess.run(["ncu", "-i", path, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(src)))[2:]
    try:
        tot = sum(int(r[2]) for r in rows)
        agg = collections.Counter()
        for r in rows:
            tok = r[1].split()
            op = tok[1] if tok and tok[0].startswith("@") else (tok[0] if tok else "?")
            agg[op] += int(r[2])
        print(f"# stall samples by SASS opcode (total {tot})")
        for op, n in agg.most_common(8):
            print(f"  {op:22s} {n:8d} {100.0 * n / tot:5.1f}%")
    except Exception as e:  # noqa: BLE001
        print("# no source page:", e)


if __name__ == "__main__":
    {"launches": launches, "kernel": kernel}[sys.argv[1]](sys.argv[2])
