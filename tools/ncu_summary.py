"""Summaries of Nsight Compute captures: (1) `ncu_summary.py rep <file.ncu-rep>...` prints the key metrics of every
captured launch from `ncu -i <rep> --page raw --csv`; (2) `ncu_summary.py launches <launches.csv>`
aggregates a `--metrics gpu__time_duration.sum` launch list by kernel (count, total, share)."""
import csv, io, subprocess, sys, collections, re

KEYS = ["launch__grid_size", "launch__block_size", "gpu__time_duration.sum", "sm__cycles_elapsed.max",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "launch__registers_per_thread", "smsp__inst_executed.sum",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "l1tex__m_xbar2l1tex_read_bytes_mem_global_op_tma_ld.sum",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]


def short(name):
    name = re.sub(r"\(.*", "", name)
    return name.replace("mivos::", "").replace("<unnamed>::", "")[-90:]


def rep(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    col = {h: i for i, h in enumerate(hdr)}
    print(f"== {path}")
    for r in rows[2:]:
        print(f"-- {short(r[col['Kernel Name']])}")
        for k in KEYS:
            if k in col:
                print(f"    {k} = {r[col[k]]} {units[col[k]]}")
        st = {h.split('smsp__average_warps_issue_stalled_')[1].split('_per_issue')[0]: r[i] for h, i in col.items()
              if h.startswith('smsp__average_warps_issue_stalled_') and h.endswith('per_issue_active.ratio')}
        top = sorted(st.items(), key=lambda kv: -float(kv[1] or 0))[:6]
        print("    stalls/issue: " + ", ".join(f"{k} {float(v):.2f}" for k, v in top))


def launches(path):
    txt = open(path).read()
    if '"ID"' not in txt:
        print(f"== {path}: no launches captured"); return
    start = txt.index('"ID"')
    rows = list(csv.DictReader(io.StringIO(txt[start:])))
    agg = collections.OrderedDict()
    total = 0.0
    for r in rows:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(r["Metric Value"].replace(",", ""))
        unit = r["Metric Unit"]
        us = v / 1e3 if unit in ("ns", "nsecond") else v * (1e3 if unit.startswith("ms") else 1.0)
        k = short(r["Kernel Name"])
        a = agg.setdefault(k, [0, 0.0])
        a[0] += 1
        a[1] += us
        total += us
    print(f"== {path}: {sum(a[0] for a in agg.values())} launches, {total/1e3:.2f} ms of kernel time (cold-cache, serialised: compare shares)")
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"  {100*us/total:5.1f} %  {us/1e3:8.2f} ms  n={n:5d}  avg {us/n:7.1f} us  {k}")


def traffic(path, key, label, out_json):
    """`ncu_summary.py traffic <rep> <fp16|tf32> <label> <out.json>`: dram__bytes_read.sum + dram__bytes_write.sum of the
    FIRST launch in the report -> out.json[key] = {bytes, launch, report} (bench.py reads it as roofline.traffic)."""
    import json, os
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, first = rows[0], rows[1], rows[2]
    col = {h: i for i, h in enumerate(hdr)}

    def to_bytes(name):
        v, u = float(first[col[name]].replace(",", "")), units[col[name]].lower()
        return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}[u]
    b = to_bytes("dram__bytes_read.sum") + to_bytes("dram__bytes_write.sum")
    d = json.load(open(out_json)) if os.path.exists(out_json) else {}
    d[key] = {"bytes": int(b), "launch": label, "kernel": short(first[col["Kernel Name"]]), "report": os.path.basename(path),
              "duration_us": float(first[col["gpu__time_duration.sum"]].replace(",", "")) * (1e-3 if units[col["gpu__time_duration.sum"]].startswith("n") else 1.0)}
    json.dump(d, open(out_json, "w"), indent=1, sort_keys=True)
    print(d[key])


if __name__ == "__main__":
    mode, files = sys.argv[1], sys.argv[2:]
    if mode == "traffic":
        traffic(*files)
    else:
        for f in files:
            rep(f) if mode == "rep" else launches(f)
