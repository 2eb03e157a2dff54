#!/usr/bin/env python
"""Summarise ncu artefacts brought back in gpurun_out/ into small text files under profiles/ (tracked).

  python tools/ncu_summary.py launches gpurun_out/launches_r1.csv profiles/launches_r1.md
  python tools/ncu_summary.py full gpurun_out/prof_conv_r1.ncu-rep profiles/conv_r1.md
"""
import csv
import subprocess
import sys
from collections import OrderedDict

METRICS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
           "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
           "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
           "launch__shared_mem_per_block_dynamic", "lts__t_bytes.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
           "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__inst_executed.sum",
           "sm__cycles_elapsed.max", "smsp__cycles_active.avg"]


def launches(src, dst):
    rows = [r for r in csv.reader(l for l in open(src) if not l.startswith("=="))]
    hdr = rows[0]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = OrderedDict()
    total = 0.0
    for r in rows[1:]:
        if len(r) <= vi:
            continue
        name = r[ki].split("(")[0].replace("void ", "").replace("b200asr::", "").replace("tc::", "")
        t = float(r[vi].replace(",", ""))
        t = t / 1e3 if r[ui] == "ns" else (t * 1e3 if r[ui] == "ms" else t)   # -> microseconds
        n, s = agg.get(name, (0, 0.0))
        agg[name] = (n + 1, s + t)
        total += t
    with open(dst, "w") as f:
        f.write("# per-launch device times (ncu --metrics gpu__time_duration.sum --clock-control none), one training step\n")
        f.write("# cold-cache, serialised: compare SHARES with bench.py's event timings, not absolutes\n")
        f.write("# source: %s ; %d launches, %.2f ms total\n\n| kernel | launches | total us | share |\n|---|---|---|---|\n" % (src, len(rows) - 1, total / 1e3))
        for name, (n, s) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write("| %s | %d | %.1f | %.1f%% |\n" % (name, n, s, 100 * s / total))
    print("wrote", dst)


def full(src, dst):
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(dst, "w") as f:
        f.write("# ncu --set full --clock-control none capture: %s\n\n" % src)
        for r in rows[2:]:
            f.write("## %s\n\n| metric | value | unit |\n|---|---|---|\n" % r[hdr.index("Kernel Name")][:110])
            for m in METRICS:
                if m in hdr:
                    i = hdr.index(m)
                    f.write("| %s | %s | %s |\n" % (m, r[i], units[i]))
            f.write("\n")
    print("wrote", dst)


def step(src, dst_md, dst_json=None):
    """One COMPLETE training step out of an `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum
    --csv` launch list of tools/one_step.py: the launches between the last two Adam kernels.  Writes the per-kernel table
    (profiles/launches_rN.md) and, if asked, profiles/ncu_traffic.json (DRAM bytes per launch per kernel and C-ABI group)."""
    import json
    import os
    rows = [r for r in csv.reader(l for l in open(src) if not l.startswith("==")) if len(r) > 5]
    hdr = rows[0]
    idi, ki, mi, vi, ui = hdr.index("ID"), hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "usecond": 1.0, "nsecond": 1e-3, "msecond": 1e3}
    launches = OrderedDict()
    for r in rows[1:]:
        d = launches.setdefault(r[idi], {"name": r[ki].split("(")[0].replace("void ", "").replace("b200asr::", "").replace("tc::", "")})
        d[r[mi]] = float(r[vi].replace(",", "")) * scale.get(r[ui], 1.0)
    seq = list(launches.values())
    adam = [i for i, d in enumerate(seq) if d["name"].startswith("adam_kernel")]
    if len(adam) >= 2:
        seq = seq[adam[-2] + 1: adam[-1] + 1]
    agg = OrderedDict()
    for d in seq:
        a = agg.setdefault(d["name"], [0, 0.0, 0.0])
        a[0] += 1
        a[1] += d.get("gpu__time_duration.sum", 0.0)
        a[2] += d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)
    total = sum(a[1] for a in agg.values())
    with open(dst_md, "w") as f:
        f.write("# one training step at cfg2 (tools/one_step.py), per-launch device times and DRAM bytes from ncu\n")
        f.write("# (--metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none): cold-cache, serialised --\n")
        f.write("# compare SHARES with bench.py's event timings, not absolutes\n")
        f.write("# source: %s ; %d launches in the step, %.2f ms total\n\n| kernel | launches | total us | share | DRAM MB / launch |\n|---|---|---|---|---|\n" % (os.path.basename(src), len(seq), total / 1e3))
        for name, (n, t, b) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write("| %s | %d | %.1f | %.1f%% | %.1f |\n" % (name, n, t, 100 * t / total, b / n / 1e6))
    print("wrote", dst_md, "(%d launches, %.2f ms)" % (len(seq), total / 1e3))
    if dst_json:
        groups = {}
        for g, subs in GROUPS.items():
            sel = [(n, t, b) for name, (n, t, b) in agg.items() if any(x in name for x in subs)]
            if sel:
                n = sum(x[0] for x in sel)
                groups[g] = {"launches": n, "dram_bytes_per_launch": sum(x[2] for x in sel) / n, "us_per_launch_under_ncu": sum(x[1] for x in sel) / n}
        git = subprocess.run(["git", "rev-parse", "--short", "HEAD"], capture_output=True, text=True, cwd=os.path.dirname(os.path.abspath(__file__))).stdout.strip()
        doc = {"git": git, "source": os.path.basename(src), "how": "ncu --clock-control none, dram__bytes_read.sum + dram__bytes_write.sum per launch, one training step of tools/one_step.py (cfg2)",
               "groups": groups, "kernels": {k: {"launches": n, "dram_bytes_per_launch": b / n, "us_per_launch_under_ncu": t / n} for k, (n, t, b) in agg.items()}}
        with open(dst_json, "w") as f:
            json.dump(doc, f, indent=1)
        print("wrote", dst_json)


# C-ABI kernel group (bench.py's roofline.kernel) -> substrings of the kernel names that implement it
GROUPS = {"conv3x3_bwd_weight": ["tc_conv3x3_wgrad"], "conv3x3_fwd": ["tc_conv3x3_halo"], "conv3x3_fwd_pool": ["tc_conv3x3_halo"], "conv3x3_bwd_data": ["tc_conv3x3_halo"],
          "linear_fwd": ["GemmPolicy<0, 0", "GemmPolicy<false, false"], "linear_bwd_data": ["GemmPolicy<0, 0", "GemmPolicy<false, false", "GemmPolicy<false, true"],
          "linear_bwd_weight": ["GemmPolicy<1, 1", "GemmPolicy<true, true"],
          "sdpa_mat_fwd": ["BGemmPolicy", "softmax_fwd"], "sdpa_mat_bwd": ["BGemmPolicy", "softmax_bwd"],
          "sdpa_fused_fwd": ["sdpa_fused_fwd"], "sdpa_fused_bwd": ["sdpa_fused_bwd"]}


def traffic(src, dst):
    """profiles/ncu_traffic.json: DRAM bytes per launch (dram__bytes_read.sum + dram__bytes_write.sum) of every kernel in an
    `ncu --set full` (or --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum) capture of bench.py,
    per kernel and per C-ABI group; bench.py reads `roofline.traffic` from it."""
    import json
    import os
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    ki, ri, wi = hdr.index("Kernel Name"), hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
    ti = hdr.index("gpu__time_duration.sum")
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    tscale = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}
    kern = OrderedDict()
    for r in rows[2:]:
        name = r[ki].split("(")[0].replace("void ", "").replace("b200asr::", "").replace("tc::", "")
        b = float(r[ri].replace(",", "")) * scale[units[ri]] + float(r[wi].replace(",", "")) * scale[units[wi]]
        t = float(r[ti].replace(",", "")) * tscale[units[ti]]
        n, sb, st = kern.get(name, (0, 0.0, 0.0))
        kern[name] = (n + 1, sb + b, st + t)
    groups = {}
    for g, subs in GROUPS.items():
        sel = [(n, sb, st) for name, (n, sb, st) in kern.items() if any(x in name for x in subs)]
        if sel:
            n = sum(x[0] for x in sel)
            groups[g] = {"launches": n, "dram_bytes_per_launch": sum(x[1] for x in sel) / n, "us_per_launch_under_ncu": sum(x[2] for x in sel) / n}
    git = subprocess.run(["git", "rev-parse", "--short", "HEAD"], capture_output=True, text=True, cwd=os.path.dirname(os.path.abspath(__file__))).stdout.strip()
    doc = {"git": git, "source": os.path.basename(src), "how": "ncu --clock-control none, dram__bytes_read.sum + dram__bytes_write.sum per launch",
           "groups": groups,
           "kernels": {k: {"launches": n, "dram_bytes_per_launch": sb / n, "us_per_launch_under_ncu": st / n} for k, (n, sb, st) in kern.items()}}
    with open(dst, "w") as f:
        json.dump(doc, f, indent=1)
    print("wrote", dst, "groups:", {g: "%.3g B" % v["dram_bytes_per_launch"] for g, v in groups.items()})


if __name__ == "__main__":
    fn = {"launches": launches, "full": full, "traffic": traffic, "step": step}[sys.argv[1]]
    fn(*sys.argv[2:])
