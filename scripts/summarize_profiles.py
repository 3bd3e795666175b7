"""Turn gpurun_out/ ncu artefacts into small tracked summaries under profiles/.
usage: python scripts/summarize_profiles.py <tag>   (e.g. r01_v1)"""
import collections, csv, os, re, subprocess, sys
tag = sys.argv[1]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G, P = os.path.join(ROOT, "gpurun_out"), os.path.join(ROOT, "profiles")
os.makedirs(P, exist_ok=True)
out = [f"# ncu summary {tag}\n"]
lc = os.path.join(G, "launches.csv")
if os.path.exists(lc):
    rows = [r for r in csv.reader(open(lc)) if len(r) > 10]
    hdr = rows[0]
    i_name, i_val = hdr.index("Kernel Name"), hdr.index("Metric Value")
    agg = collections.OrderedDict()
    for r in rows[1:]:
        a = agg.setdefault(re.sub(r"\(.*", "", r[i_name]), [0, 0.0])
        a[0] += 1
        a[1] += float(r[i_val].replace(",", "")) / 1e6
    tot = sum(a[1] for a in agg.values())
    out.append("## launch list (`ncu --metrics gpu__time_duration.sum --clock-control none`, cold-cache serialised: compare SHARES)\n")
    out.append(f"command: `python bench.py --steps 1 --warmup 1 --rays 8192 --ray-batch 8192 --no-cpu-baseline {os.environ.get('BENCH_EXTRA','')}`; "
               f"{len(rows)-1} launches captured, {tot:.1f} ms total\n")
    out.append("| kernel | launches | total ms | share |\n|---|---|---|---|")
    for n, (c, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:12]:
        out.append(f"| `{n[:80]}` | {c} | {ms:.2f} | {100*ms/tot:.2f}% |")
    out.append("")
rep = os.path.join(G, "prof.ncu-rep")
if os.path.exists(rep):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    want = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
            "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
            "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
            "lts__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
            "l1tex__data_pipe_lsu_wavefronts.sum.pct_of_peak_sustained_elapsed", "l1tex__t_sector_hit_rate.pct",
            "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
            "l1tex__t_requests_pipe_lsu_mem_global_op_red.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum",
            "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__inst_executed.sum",
            "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
            "smsp__issue_active.avg.pct_of_peak_sustained_active",
            "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
            "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
            "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
            "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
            "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio"]
    kn = idx["Kernel Name"]
    # dram bytes per launch of every kernel -> profiles/ncu_traffic.json (bench.py's roofline.traffic)
    import json
    traffic = {}
    for r in rows[2:]:
        name = re.sub(r"[<(].*", "", r[kn]).replace("void ", "").strip()
        tot = 0.0
        for m in ("dram__bytes_read.sum", "dram__bytes_write.sum"):
            mult = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}[units[idx[m]]]
            tot += float(r[idx[m]].replace(",", "")) * mult
        traffic.setdefault(name, tot)
    rays_per_launch = int(os.environ.get("PROFILE_RAYS", "8192"))
    json.dump({"source": f"{tag}_ncu_summary.md", "config": f"L=16, {rays_per_launch} rays x 768 samples per launch",
               "rays_per_launch": rays_per_launch, "dram_bytes_per_launch": traffic},
              open(os.path.join(P, "ncu_traffic.json"), "w"), indent=1)
    # which unit binds each kernel (bench.py quotes these next to its live timings)
    units_pct = {"l1tex_lsu_data_pipe_pct": "l1tex__data_pipe_lsu_wavefronts.sum.pct_of_peak_sustained_elapsed",
                 "l2_throughput_pct": "lts__throughput.avg.pct_of_peak_sustained_elapsed",
                 "dram_throughput_pct": "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
                 "tensor_pipe_pct": "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
                 "fma_pipe_pct": "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
                 "issue_active_pct": "smsp__issue_active.avg.pct_of_peak_sustained_active",
                 "warps_active_pct": "sm__warps_active.avg.pct_of_peak_sustained_active"}
    binding = {}
    for r in rows[2:]:
        name = re.sub(r"[<(].*", "", r[kn]).replace("void ", "").strip()
        if name in binding:
            continue
        d = {}
        for k, m in units_pct.items():
            if m in idx:
                try:
                    d[k] = float(r[idx[m]].replace(",", ""))
                except ValueError:
                    pass
        pipes = {k: v for k, v in d.items() if k in ("l1tex_lsu_data_pipe_pct", "l2_throughput_pct", "dram_throughput_pct", "tensor_pipe_pct", "fma_pipe_pct")}
        if pipes:
            top = max(pipes, key=pipes.get)
            d["limiter"] = f"{top} = {pipes[top]:.0f} % of peak (ncu --set full, {tag})"
            d["limiter_unit"] = {"l1tex_lsu_data_pipe_pct": "L1TEX LSU data pipe (wavefronts)", "l2_throughput_pct": "L2 (lts) throughput",
                                 "dram_throughput_pct": "DRAM (HBM) throughput", "tensor_pipe_pct": "tensor pipe",
                                 "fma_pipe_pct": "FP32 FMA pipe"}[top]
            d["limiter_pct"] = pipes[top]
        binding[name] = d
    json.dump({"source": f"{tag}_ncu_summary.md", "kernels": binding}, open(os.path.join(P, "ncu_binding.json"), "w"), indent=1)
    out.append("## `ncu --set full --clock-control none --import-source on` capture (per launch)\n")
    out.append("| metric | " + " | ".join(re.sub(r"\(.*", "", r[kn]) for r in rows[2:]) + " | unit |")
    out.append("|---|" + "---|" * (len(rows) - 1))
    for w in want:
        if w in idx:
            out.append(f"| {w} | " + " | ".join(r[idx[w]] for r in rows[2:]) + f" | {units[idx[w]]} |")
    out.append("")
for f in ("probe.log",):
    p = os.path.join(G, f)
    if os.path.exists(p):
        out.append(f"## {f} (CUDA-event timings, not under a profiler)\n```")
        out += [l.rstrip() for l in open(p) if "[probe]" in l]
        out.append("```")
open(os.path.join(P, f"{tag}_ncu_summary.md"), "w").write("\n".join(out) + "\n")
print("\n".join(out))
