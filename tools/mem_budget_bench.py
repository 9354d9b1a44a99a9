"""Throughput of mapping within a device-memory budget (mpb_ctx_set_mem_budget).

C2 (default): the C2 set through mpb_map_file on one context in automatic mode and at explicit budgets; per run proteins/s, the
slices of each stage, the peak the arenas held, the phase walls, and whether the PAF is the automatic mode's byte for byte.
--config C3: the full 3 Gbp set with -I through one context at the default -K (automatic mode, or --budget), with its peak, proteins/s
and the PAF's sha256 against the reference CLI's (tools/parity.py machinery).  --config C3s: the same on the 1 Gbp cut of it.

Rows go to results/h100_mem_budget.jsonl (--out), each with the device name and its power limit."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import miniprot_b200 as mp  # noqa: E402
from miniprot_b200 import synth  # noqa: E402

MEM_FIELDS = ("budget", "peak_held", "n_slices_seed", "n_slices_refine", "n_subwaves", "n_released", "bytes_released", "n_over_budget")


def device():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=60)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return {"device": name, "power_limit": power}
    except Exception:  # noqa: BLE001 -- a label, not a gate
        return {"device": "unknown", "power_limit": "unknown"}


def parse_size(s: str) -> int:
    m = {"k": 10, "m": 20, "g": 30}
    return int(s[:-1]) << m[s[-1].lower()] if s[-1].lower() in m else int(s)


def run(ctx, mi, p, out, mo, budget):
    ctx.set_mem_budget(budget)
    ctx.reset_stats()
    t0 = time.time()
    mp.map_file(ctx, mi, p, out, mo)
    dt = time.time() - t0
    st, ms = ctx.stats(), ctx.mem_stats()
    return dt, st, ms


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--config", default="C2", choices=["C2", "C3", "C3s"])
    ap.add_argument("--budgets", default="16g,4g,1g,256m", help="explicit budgets of the C2 runs (after one in automatic mode)")
    ap.add_argument("--budget", default="0", help="budgets of the C3 / C3s runs, comma-separated (0: automatic)")
    ap.add_argument("--repeat", type=int, default=3, help="C2: runs per budget (the fastest is reported, and the range of all)")
    ap.add_argument("--dir", default=os.environ.get("MPB_BENCH_DIR", "/tmp/mpb_bench"))
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_mem_budget.jsonl"))
    a = ap.parse_args()
    dev = device()
    d = os.path.join(a.dir, a.config)
    rows = []
    if a.config == "C2":
        g, p = synth.generate(synth.CONFIGS["C2"], d)
        n_prot = sum(1 for line in open(p) if line.startswith(">"))
        mi = mp.idx_load(g, os.cpu_count() or 8)
        ctx = mp.Context(0)
        mo = mp.mapopt()
        base = None
        for b in [0] + [parse_size(x) for x in a.budgets.split(",") if x]:
            best, dts = None, []
            for _ in range(a.repeat):
                out = os.path.join(d, "budget.paf")
                dt, st, ms = run(ctx, mi, p, out, mo, b)
                dts.append(dt)
                if best is None or dt < best[0]:
                    best = (dt, st, ms)
            digest = hashlib.sha256(open(out, "rb").read()).hexdigest()
            base = base or digest
            dt, st, ms = best
            row = {"config": "C2", "timed": "mpb_map_file, file reading and PAF writing included", "proteins_per_s": round(n_prot / dt, 1),
                   "proteins_per_s_range": [round(n_prot / max(dts), 1), round(n_prot / min(dts), 1)], "wall_s": round(dt, 3), "identical_to_auto": digest == base,
                   **{f: getattr(ms, f) for f in MEM_FIELDS}, "ms_wall": [round(x, 1) for x in st.ms_wall], **dev}
            print(json.dumps(row), flush=True)
            rows.append(row)
        ctx.close()
        mp.lib().mp_idx_destroy(mi)
    else:
        import parity

        for b in [parse_size(x) for x in a.budget.split(",") if x]:
            ctx = mp.Context(0)
            ctx.set_mem_budget(b)
            r = parity.run_config(a.config, ["-I"], d, os.cpu_count() or 8, ctx=ctx)[0]
            ms = ctx.mem_stats()
            row = {"config": a.config, "opt": "-I", "identical_to_reference": r["identical"], "sha256": r["sha256_ours"], "sha256_ref": r["sha256_ref"],
                   "proteins_per_s": round(r["n_proteins"] / r["ours_s"], 1), "wall_s": r["ours_s"], **{f: getattr(ms, f) for f in MEM_FIELDS},
                   "ms_wall": r["wall_ms"], **dev}
            print(json.dumps(row), flush=True)
            rows.append(row)
            ctx.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "a") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    return 0 if all(r.get("identical_to_auto", r.get("identical_to_reference")) for r in rows) else 1


if __name__ == "__main__":
    sys.exit(main())
