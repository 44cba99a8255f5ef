#!/usr/bin/env python
"""Turns the raw outputs of tools/profile_round.sh into summaries under profiles/ (kept out of git: they describe the build
and the GPU they were captured on):
  launches_<tag>.csv / launches_<tag>_summary.txt   per-kernel share of a bench step (ncu gpu__time_duration pass)
  ncu_<tag>.json                                     key metrics of the full captures (one launch per hot kernel)
  sass_mix_<tag>.txt                                 SASS opcode mix (executed warp instructions) + hottest source lines per kernel
  traffic_<tag>.json                                 DRAM bytes per launch of the hot kernels
  bench_<tag>.json                                   the bench line of the same GPU
Needs the `ncu`, `cuobjdump`, `nvdisasm` CLIs (reads .ncu-rep files; no GPU).  Usage: python tools/summarize_profiles.py r02"""
import collections, csv, io, json, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "gpurun_out"); P = os.path.join(ROOT, "profiles")
TAG = sys.argv[1] if len(sys.argv) > 1 else "r02"
KERNELS = {"k_walk": ("final_k_walk.ncu-rep", "_ZN3pgs6k_walk"), "k_emit": ("final_k_emit.ncu-rep", "_ZN3pgs6k_emit"),
           "k_get": ("final_k_get.ncu-rep", "_ZN3pgs5k_get"), "k_scan_fwd": ("final_k_scan_fwd.ncu-rep", "_ZN3pgs10k_scan_fwd")}
STEM = {"k_walk": "compact", "k_emit": "compact", "k_get": "lookup", "k_scan_fwd": "lookup"}
KEEP = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "launch__shared_mem_per_block_dynamic", "launch__grid_size", "launch__block_size",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "dram__throughput.avg.pct_of_peak_sustained_elapsed"]
SCALE = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1}


def raw(rep):
    out = subprocess.check_output(["ncu", "-i", rep, "--page", "raw", "--csv"], stderr=subprocess.DEVNULL).decode()
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, r = rows[0], rows[1], rows[2]
    d = {k: {"unit": units[hdr.index(k)], "value": r[hdr.index(k)]} for k in KEEP if k in hdr}
    d["kernel"] = r[hdr.index("Kernel Name")]
    return d


def sass_mix(rep, kpref, stem, so):
    os.system(f"rm -rf /tmp/xelf && mkdir -p /tmp/xelf && cd /tmp/xelf && cuobjdump -xelf all {so} >/dev/null 2>&1")
    cub = [f for f in os.listdir("/tmp/xelf") if f.startswith(stem) and f.endswith(".cubin")][0]
    sass = subprocess.check_output(["nvdisasm", "-g", "-c", os.path.join("/tmp/xelf", cub)]).decode().split("\n")
    starts = [i for i, l in enumerate(sass) if l.startswith(kpref) and l.rstrip().endswith(":")]
    out = subprocess.check_output(["ncu", "-i", rep, "--page", "source", "--csv"], stderr=subprocess.DEVNULL).decode()
    rows = list(csv.reader(out.split("\n")))
    hdr = rows[1]
    data = [r for r in rows[2:] if len(r) == len(hdr)]
    ix, isrc = hdr.index("Instructions Executed"), hdr.index("Source")
    ops = collections.Counter()
    for d in data:
        m = re.match(r"\s*(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", d[isrc])
        if m: ops[m.group(1).split(".")[0]] += int(d[ix])
    lines = collections.Counter()
    for start in starts:  # the instantiation whose instruction count matches the capture
        end = next((i for i in range(start + 1, len(sass)) if sass[i].startswith("//--------------------- .text.")), len(sass))
        insts, cur = [], None
        for l in sass[start:end]:
            m = re.match(r'\s*//## File "([^"]+)", line (\d+)', l)
            if m: cur = (os.path.basename(m.group(1)), int(m.group(2))); continue
            if re.match(r"\s*/\*[0-9a-f]{4,6}\*/\s+\S", l): insts.append(cur)
        if len(insts) == len(data):
            for c, d in zip(insts, data): lines[c] += int(d[ix])
            break
    return ops, lines


def main():
    # 1. launch list
    src = os.path.join(G, "final_launches.csv")
    if os.path.exists(src):
        text = [l for l in open(src) if not l.startswith("==")]
        open(os.path.join(P, f"launches_{TAG}.csv"), "w").writelines(text)
        agg = collections.OrderedDict()
        for r in csv.DictReader(io.StringIO("".join(text))):
            if r.get("Metric Name") != "gpu__time_duration.sum": continue
            v = float(r["Metric Value"].replace(",", "")); u = r["Metric Unit"]
            ms = v / 1e6 if u in ("ns", "nsecond") else v / 1e3 if u in ("us", "usecond") else v
            a = agg.setdefault(r["Kernel Name"].split("(")[0], [0, 0.0]); a[0] += 1; a[1] += ms
        tot = sum(a[1] for a in agg.values())
        with open(os.path.join(P, f"launches_{TAG}_summary.txt"), "w") as f:
            f.write("ncu --metrics gpu__time_duration.sum --clock-control none; command: python bench.py --steps 2 --warmup 1 --skip-cpu --skip-e2e "
                    "--skip-sharded --skip-sweep --skip-ycsb\n(cold-cache, serialised launches: compare shares, not absolutes)\n")
            for k, (n, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
                f.write(f"{k:70s} launches {n:4d}  total {ms:9.3f} ms  share {100*ms/tot:5.1f}%\n")
        print(open(os.path.join(P, f"launches_{TAG}_summary.txt")).read())
    # 2. full captures, traffic, SASS mix
    caps, traffic = {}, {}
    so = os.path.join(G, "lib_at_profile.so")
    with open(os.path.join(P, f"sass_mix_{TAG}.txt"), "w") as mix:
        mix.write("SASS opcode mix of the full-size launches (executed warp instructions, ncu source page) and the hottest source lines\n")
        for name, (rep, kpref) in KERNELS.items():
            pth = os.path.join(G, rep)
            if not os.path.exists(pth): continue
            d = raw(pth)
            caps[name] = d
            rd = float(d["dram__bytes_read.sum"]["value"].replace(",", "")) * SCALE[d["dram__bytes_read.sum"]["unit"]]
            wr = float(d["dram__bytes_write.sum"]["value"].replace(",", "")) * SCALE[d["dram__bytes_write.sum"]["unit"]]
            traffic[name] = {"dram_bytes_per_launch": int(rd + wr), "dram_read_bytes": int(rd), "dram_write_bytes": int(wr),
                             "source": f"ncu --set full capture of one launch at the bench size (profiles/ncu_{TAG}.json)"}
            ops, lines = sass_mix(pth, kpref, STEM[name], so)
            tot = sum(ops.values()) or 1
            mix.write(f"\n== {name}: {d['kernel'][:90]}\n   {tot} warp instructions, {d['gpu__time_duration.sum']['value']} {d['gpu__time_duration.sum']['unit']} under ncu\n")
            groups = collections.Counter()
            for o, n in ops.items():
                g = ("global/local memory" if o in ("LDG", "STG", "LD", "ST", "LDL", "STL", "RED", "ATOMG", "ATOM", "LDGSTS", "UBLKCP", "LDGDEPBAR", "DEPBAR") else
                     "shared memory" if o in ("LDS", "STS", "ATOMS", "LDSM") else
                     "warp collectives" if o in ("SHFL", "VOTE", "VOTEU", "MATCH", "REDUX", "WARPSYNC", "BAR") else
                     "control flow" if o in ("BRA", "BSSY", "BSYNC", "BREAK", "EXIT", "CALL", "RET", "NOP", "BMOV", "WARPSYNC") else
                     "integer / logic / move")
                groups[g] += n
            for g, n in groups.most_common(): mix.write(f"   {g:26s} {100*n/tot:5.1f}%\n")
            mix.write("   top opcodes: " + ", ".join(f"{o} {100*n/tot:.1f}%" for o, n in ops.most_common(14)) + "\n")
            lt = sum(lines.values()) or 1
            for c, n in lines.most_common(8):
                if c: mix.write(f"   {100*n/lt:5.1f}%  {c[0]}:{c[1]}\n")
    json.dump({"note": "ncu --set full --clock-control none captures at the full bench size (4 x 2.5M records; reads: 262144 gets / 16384 "
                       "prefix scans); times under ncu replay are not bench values", "captures": caps},
              open(os.path.join(P, f"ncu_{TAG}.json"), "w"), indent=1)
    if traffic: json.dump(traffic, open(os.path.join(P, f"traffic_{TAG}.json"), "w"), indent=1)
    if os.path.exists(os.path.join(G, "final_bench.json")):
        open(os.path.join(P, f"bench_{TAG}.json"), "w").write(open(os.path.join(G, "final_bench.json")).read())
    print(open(os.path.join(P, f"sass_mix_{TAG}.txt")).read())


if __name__ == "__main__":
    main()
