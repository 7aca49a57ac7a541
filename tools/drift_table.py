"""Markdown table of the full-size parity runs: reads the drift curves tests/test_gpu_zzz_fullsize.py writes
($MIVOS_DRIFT_DIR/drift_*.json) and prints one row per case.  Usage: python tools/drift_table.py DIR > table.md"""
import glob
import json
import os
import sys

d = sys.argv[1]
print("| case | max dp | mean dp | last-frame max dp | mask mismatch worst frame | last frame | decided pixels (mismatching) | max dp per quarter of the clip |")
print("|---|---|---|---|---|---|---|---|")
for p in sorted(glob.glob(os.path.join(d, "drift_*.json"))):
    r = json.load(open(p))
    name = os.path.basename(p)[len("drift_"):-len(".json")]
    per = r["dp_max_per_frame"]
    q = max(1, len(per) // 4)
    quarters = " ".join(f"{max(per[i * q:(i + 1) * q if i < 3 else len(per)]):.1e}" for i in range(4))
    dec = r["decided_pixels_grid"] + r["decided_pixels_last"]
    dm = r["decided_mismatch_grid"] + r["decided_mismatch_last"]
    print(f"| {name} | {r['dp_max']:.2e} | {r['dp_mean']:.1e} | {r['last_dp_max']:.2e} | {r['mask_mismatch_max']:.2e} | "
          f"{r['last_mask_mismatch']:.2e} | {dec} ({dm}) | {quarters} |")
