"""Turns gpurun_out/ artefacts into the tracked summaries under profiles/ (round-tagged).
   python tools/summarize_profiles.py <tag> <launches.csv> <prof.ncu-rep> <bench.json> [<bench_ref.json>]"""
import collections, csv, json, os, subprocess, sys
tag, launches, rep, bench = sys.argv[1:5]
ref = sys.argv[5] if len(sys.argv) > 5 else None
out = [f"# {tag}: ncu + bench summary (H100, sm_90a)\n"]
j = json.load(open(bench))
out.append("## bench.py line (N=1)\n```json\n" + json.dumps(j, indent=1)[:6000] + "\n```\n")
if ref and os.path.exists(ref):
    out.append("## bench.py --impl reference line\n```json\n" + open(ref).read().strip()[:3000] + "\n```\n")
rows = list(csv.reader(open(launches)))
hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
hdr = rows[hi]; kn, mv, mu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
agg = collections.OrderedDict()
for r in rows[hi + 1:]:
    if len(r) <= mv: continue
    v = float(r[mv].replace(",", "")); u = r[mu]
    v = v / 1e3 if u == "us" else v / 1e6 if u == "ns" else v * 1e3 if u in ("s", "second") else v
    name = r[kn].split("(")[0]
    a = agg.setdefault(name, [0, 0.0]); a[0] += 1; a[1] += v
tot = sum(v[1] for v in agg.values())
out.append("## launch list (ncu --metrics gpu__time_duration.sum, same bench command; cold-cache, serialised: compare shares)\n")
out.append("| kernel | launches | total ms | share |\n|---|---|---|---|")
for k, (c, v) in agg.items():
    out.append(f"| `{k[-70:]}` | {c} | {v:.3f} | {100 * v / tot:.1f}% |")
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rr = list(csv.reader(raw.splitlines())); hdr, units = rr[0], rr[1]
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "l1tex__m_xbar2l1tex_read_bytes.sum",
        "lts__t_sectors_srcunit_tex_op_read.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "launch__registers_per_thread",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "launch__shared_mem_per_block_dynamic", "lts__t_sector_hit_rate.pct",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warp_latency_per_inst_issued.ratio"]
out.append("\n## ncu --set full, den kernels (bench.py --T 100: one launch = 100 frames of N=64; traffic scales with T)\n")
for r in rr[2:]:
    out.append(f"### `{r[hdr.index('Kernel Name')][:90]}`\n| metric | value | unit |\n|---|---|---|")
    for w in want:
        if w in hdr:
            i = hdr.index(w); out.append(f"| {w} | {r[i]} | {units[i]} |")
    out.append("")
# per-launch DRAM traffic of the den kernels, per frame (the capture ran bench.py --T 100 => 100 frames per launch)
traffic = {}
for r in rr[2:]:
    name = r[hdr.index("Kernel Name")]
    key = "den_forward_kernel" if "den_forward" in name else "den_backward_kernel" if "den_backward" in name else None
    if not key: continue
    def val(m):
        i = hdr.index(m); v = float(r[i].replace(",", "")); u = units[i].lower()
        return v * (1e9 if u.startswith("gbyte") else 1e6 if u.startswith("mbyte") else 1e3 if u.startswith("kbyte") else 1)
    def pct(m):
        return float(r[hdr.index(m)].replace(",", "")) if m in hdr else None
    traffic[key] = {"dram_bytes_per_frame": (val("dram__bytes_read.sum") + val("dram__bytes_write.sum")) / 100.0,
                    "l2_to_sm_bytes_per_frame": val("l1tex__m_xbar2l1tex_read_bytes.sum") / 100.0 if "l1tex__m_xbar2l1tex_read_bytes.sum" in hdr else None,
                    "pipe_fma_pct": pct("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active"),
                    "pipe_xu_pct": pct("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active"),
                    "issue_active_pct": pct("smsp__issue_active.avg.pct_of_peak_sustained_active"),
                    "capture": f"{tag}: ncu --set full, bench.py --T 100 (N=64, V=218, 1M-arc graph)"}
json.dump(traffic, open("profiles/traffic.json", "w"), indent=1)
os.makedirs("profiles", exist_ok=True)
open(f"profiles/{tag}_summary.md", "w").write("\n".join(out) + "\n")
print("wrote", f"profiles/{tag}_summary.md")
import shutil
shutil.copyfile(launches, f"profiles/{tag}_launches.csv")   # the launch list the summary table was made from
