#!/usr/bin/env python
"""Durations of the fronts that do not fit in shared memory and run on ONE CTA (a team of one on the team code,
task word G = 1, or cta_front's HBM mode, G = 0), from k_factor traces written by
`tools/panel_trace.py --dump-trace`: children ready -> eliminated per front, their sum and median, the fronts of
the traced critical path, and a least-squares fit of the HBM mode's duration model (plan.c: front_lat_us).

    python tools/solo_trace.py before.npz [after.npz ...]
"""
import sys

import numpy as np
from scipy.optimize import nnls


def fits_smem(m):
    ld = (m + 2) // 2 * 2
    return ld * m + (ld + 1) // 2 + 2 <= 25600


def report(path):
    z = np.load(path)
    tf, tasks, nwait = z["tf"].astype(np.int64), z["tasks"], z["nwait"].astype(np.int64)
    m, c, parent = 3 * z["mb"].astype(np.int64), 3 * z["cb"].astype(np.int64), z["parent"]
    G = (nwait >> 24) & 0x7F
    first = ((nwait >> 16) & 0xFF) == 0
    row = {int(s): k for k, s in enumerate(tasks) if first[k]}
    dur = {s: (tf[k, 5] - tf[k, 2]) / 1e3 for s, k in row.items()}
    one = [s for s, k in row.items() if G[k] <= 1 and not fits_smem(int(m[s]))]
    d1 = np.array([dur[s] for s in one])
    print(f"{path}: k_factor {float(z['kernel_ms'][1]):.3f} ms; {len(one)} one-CTA fronts in HBM "
          f"(G = {sorted(set(int(G[row[s]]) for s in one))}): sum {d1.sum() / 1e3:.2f} CTA-ms, median {np.median(d1):.1f} us")
    # the traced critical path: from the front that finishes last, down through the child that finished last
    kids = {}
    for s in row:
        if parent[s] >= 0:
            kids.setdefault(int(parent[s]), []).append(s)
    s = max(row, key=lambda x: tf[row[x], 5])
    path = []
    while s is not None:
        path.append(s)
        ks = kids.get(s, [])
        s = max(ks, key=lambda x: tf[row[x], 5]) if ks else None
    on = [x for x in path if x in set(one)]
    span = (tf[row[path[0]], 5] - tf[row[path[-1]], 2]) / 1e3
    print(f"  critical path: {len(path)} fronts, {span:.0f} us; one-CTA fronts on it: {len(on)}, "
          f"{sum(dur[x] for x in on):.0f} us" + (f", worst sn {max(on, key=dur.get)} (m {m[max(on, key=dur.get)]}, "
                                               f"c {c[max(on, key=dur.get)]}) {max(dur[x] for x in on):.0f} us" if on else ""))
    solo = [s for s in one if G[row[s]] == 0]
    if len(solo) >= 8:
        mm, cc, y = (np.array([m[s] for s in solo], float), np.array([c[s] for s in solo], float),
                     np.array([dur[s] for s in solo]))
        A = np.c_[np.ones_like(mm), mm, cc, cc * mm]
        coef, _ = nnls(A, y)
        err = np.abs(A @ coef - y) / y
        print(f"  HBM-mode model a + b*m + c*c + d*c*m: {', '.join(f'{v:.4g}' for v in coef)}; "
              f"median error {100 * np.median(err):.0f} %, 90th percentile {100 * np.percentile(err, 90):.0f} %")


if __name__ == "__main__":
    for p in sys.argv[1:]:
        report(p)
