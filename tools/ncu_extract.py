#!/usr/bin/env python
"""profiles/ncu_traffic.json from the raw exports of the ncu --set full captures (no GPU needed).

    ncu -i gpurun_out/X_100k_batch_prof.ncu-rep --page raw --csv > profiles/X_100k_batch_prof_raw.csv   (same for m3500)
    python tools/ncu_extract.py profiles/X_100k_batch_prof_raw.csv profiles/X_m3500_batch_prof_raw.csv
"""
import csv
import os
import json
import sys

MULT = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}


def main():
    out = {"_comment": "dram__bytes_read.sum + dram__bytes_write.sum per launch of the solve kernels, from the ncu --set full "
                       "captures named in 'source' (bench.py copies them into roofline_kernels[].traffic)"}
    for wl, f in zip(("manhattan_batch", "m3500_batch"), sys.argv[1:3]):
        rows = list(csv.reader(open(f)))
        hdr, units = rows[0], rows[1]
        ir, iw, ik = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum"), hdr.index("Kernel Name")
        agg = {}
        for r in rows[2:]:
            k = r[ik].split("(")[0]
            agg[k] = agg.get(k, 0) + float(r[ir]) * MULT[units[ir]] + float(r[iw]) * MULT[units[iw]]
        out[wl] = {"source": f, "k_linearize": {"bytes": int(agg.get("k_linearize", 0))},
                   "k_factor": {"bytes": int(agg.get("k_factor", 0) + agg.get("k_factor_leaf", 0)), "note": "k_factor + k_factor_leaf"},
                   "k_backsolve": {"bytes": int(agg.get("k_backsolve", 0) + agg.get("k_backsolve_leaf", 0)),
                                   "note": "k_backsolve + k_backsolve_leaf"}}
    os.makedirs("profiles", exist_ok=True)
    json.dump(out, open("profiles/ncu_traffic.json", "w"), indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
