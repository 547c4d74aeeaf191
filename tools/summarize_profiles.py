#!/usr/bin/env python
"""Turns the ncu captures in gpurun_out/ into the small text summaries committed under profiles/.
usage: summarize_profiles.py TAG   (reads gpurun_out/TAG_*.ncu-rep, gpurun_out/TAG_launches.csv)"""
import csv, io, os, subprocess, sys, collections

tag = sys.argv[1] if len(sys.argv) > 1 else "r1"
G, P = "gpurun_out", "profiles"
os.makedirs(P, exist_ok=True)
WANT = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static", "launch__waves_per_multiprocessor",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "smsp__inst_executed.sum"]


def raw(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    return rows[0], rows[1], rows[2:]


for name in ("inflate", "rans", "bam", "tok3", "fast32", "tile4", "cram_records"):
    rep = os.path.join(G, "%s_%s.ncu-rep" % (tag, name))
    if not os.path.exists(rep):
        continue
    hdr, units, rows = raw(rep)
    with open(os.path.join(P, "%s_%s_ncu_summary.txt" % (tag, name)), "w") as f:
        f.write("# ncu --set full --clock-control none, one launch per row; from %s\n" % os.path.basename(rep))
        for r in rows:
            f.write("\nkernel: %s\n" % r[hdr.index("Kernel Name")][:110])
            for k in WANT:
                if k in hdr:
                    f.write("  %-82s %s %s\n" % (k, r[hdr.index(k)], units[hdr.index(k)]))
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--print-source", "cuda,sass", "--csv"], capture_output=True, text=True).stdout
    if "Line No" in src:
        tmp = "/tmp/_src_%s.csv" % name
        open(tmp, "w").write(src)
        lines = subprocess.run([sys.executable, "tools/ncu_lines.py", tmp, "1"], capture_output=True, text=True).stdout
        with open(os.path.join(P, "%s_%s_source_lines.txt" % (tag, name)), "w") as f:
            f.write("# share of executed warp instructions / stall samples per CUDA source line (top 50)\n" + lines)

lc = os.path.join(G, "%s_launches.csv" % tag)
if os.path.exists(lc):
    agg = collections.OrderedDict()
    rows = [r for r in csv.reader(open(lc)) if len(r) > 5 and r[0].isdigit()]
    for r in rows:
        k = r[4][:100]
        try: t = float(r[-1].replace(",", ""))
        except ValueError: continue
        a = agg.setdefault(k, [0, 0.0]); a[0] += 1; a[1] += t
    tot = sum(v[1] for v in agg.values())
    with open(os.path.join(P, "%s_launch_list.txt" % tag), "w") as f:
        f.write("# ncu --metrics gpu__time_duration.sum --clock-control none over `bench.py --gb 1 --steps 2 --warmup 1` (cold-cache, serialised: compare shares)\n")
        f.write("# launches   total_ns   share   kernel\n")
        for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write("%6d %14.0f %6.2f%%  %s\n" % (n, t, 100 * t / tot, k))
    subprocess.run(["cp", lc, os.path.join(P, "%s_launches.csv" % tag)])
print("done")
