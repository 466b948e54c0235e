#!/usr/bin/env python
"""tools/cta_tail.py -- how evenly the C = 32 tensor-core step kernel's CTAs finish on bench.py's pair8 step.

Needs a library built with the per-CTA clocks of sfm_step_tc_kernel (every code size records them):
    tools/build_variant.sh clocks "-DDFK_EXP_CTA_CLOCKS"
    DFK_LIB=tools/variants/libdfk_clocks.so python tools/cta_tail.py [--launches N] [--json OUT]

Every CTA records %globaltimer at entry and exit, its tile count and its count of tiles with a valid pixel.  Per launch,
times are taken from the earliest CTA entry; the kernel span is the latest CTA exit.  Printed (median over the launches):
the median, p99 and max CTA finish time, the tail (max - median finish) as a share of the span, and the spread of the
per-CTA valid-tile counts.  The inputs are bench.py's pair8 step (8 distinct pairs x 4 levels, seed 0).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pair8_work(al, torch, dev):
    import numpy as np

    from bench import CS, H0, LEVELS, W0
    from deepfactors_b200 import synth
    base = synth.make_pair(W0, H0, CS, LEVELS, seed=0)
    base_dev = [{k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in dict(
        img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1).items()} for L in base.levels]
    items = []
    for q in range(8):  # bench.py variant(l, q): every pair owns all of its buffers
        for l, L in enumerate(base.levels):
            d = dict(base_dev[l])
            if q > 0:
                d["prx0_jac"] = torch.roll(d["prx0_jac"], shifts=(3 * q, 5 * q), dims=(0, 1)).contiguous()
                d["img0"] = (d["img0"] * (1.0 - 0.01 * (q % 50))).contiguous()
                for k in ("img1", "grad1", "dpt0"):
                    d[k] = d[k].clone()
            d["valid0"] = torch.zeros_like(d["img0"])
            items.append(dict(pose0=base.pose0, pose1=base.pose1, cam=L.cam, **d))
    return al.make_work_items(items), items


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=30)
    ap.add_argument("--json", default=None, help="also write the per-launch statistics and the last launch's CTAs here")
    args = ap.parse_args()

    import numpy as np
    import torch

    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner
    lib = _lib.lib()
    if not hasattr(lib, "dfk_exp_cta_clocks"):
        sys.exit("cta_tail.py: the library has no per-CTA clocks; build it with -DDFK_EXP_CTA_CLOCKS and load it with DFK_LIB")
    lib.dfk_exp_cta_clocks.argtypes = [C.c_void_p, C.c_int]
    lib.dfk_exp_cta_clocks.restype = C.c_int

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    al = SfmAligner(32, gram_mode="tf32x3")
    work, items = pair8_work(al, torch, dev)
    records = torch.zeros((len(items), _lib.record_floats(32)), dtype=torch.float32, device=dev)
    for _ in range(5):
        al.RunStepBatch(work, records)
    torch.cuda.synchronize()

    # every launch of the same work list has the same grid: its CTAs are the leading records with an exit time
    n_max = 8192
    buf = np.zeros((n_max, 4), dtype=np.uint64)
    stats = []
    for _ in range(args.launches):
        al.RunStepBatch(work, records)
        if lib.dfk_exp_cta_clocks(buf.ctypes.data, n_max) != 0:
            sys.exit("cta_tail.py: dfk_exp_cta_clocks failed")
        live = buf[:, 1] > 0
        ctas = int(live.sum())
        b = buf[:ctas].astype(np.int64)
        t0 = b[:, 0].min()
        start, end = (b[:, 0] - t0) / 1e3, (b[:, 1] - t0) / 1e3  # us
        tiles, valid = b[:, 2] >> 32, b[:, 2] & 0xffffffff
        span = end.max()
        med = float(np.median(end))
        stats.append(dict(ctas=ctas, span_us=float(span), start_max_us=float(start.max()), finish_median_us=med,
                          finish_p99_us=float(np.percentile(end, 99)), finish_max_us=float(span),
                          finish_min_us=float(end.min()), tail_share=float((span - med) / span),
                          max_over_median=float(span / med),
                          tiles_min=int(tiles.min()), tiles_max=int(tiles.max()),
                          valid_tiles_mean=float(valid.mean()), valid_tiles_std=float(valid.std()),
                          valid_tiles_min=int(valid.min()), valid_tiles_max=int(valid.max()),
                          sms=int(len(np.unique(b[:, 3])))))
    keys = [k for k in stats[0] if k not in ("ctas", "sms")]
    summary = {"ctas": stats[-1]["ctas"], "sms": stats[-1]["sms"], "launches": args.launches,
               "device": torch.cuda.get_device_name(0)}
    for k in keys:
        v = np.array([s[k] for s in stats], dtype=np.float64)
        summary[k] = float(np.median(v))
        summary[k + "_range"] = [float(v.min()), float(v.max())]
    print(json.dumps(summary))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"summary": summary, "launches": stats,
                       "last_launch_ctas": b.tolist(), "columns": "entry_ns, exit_ns, tiles<<32|valid_tiles, smid"}, f)


if __name__ == "__main__":
    main()
