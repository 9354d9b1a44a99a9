"""Time of the k-mer index build on the device within a device-memory budget (mpb_ctx_set_mem_budget on the default context, which
mp_idx_load builds on).

For each genome (synthetic C2, C3s and, with --configs C3, the full 3 Gbp set), mp_idx_load from FASTA runs in automatic mode and
at each explicit budget, --repeat times with the budgets alternating.  Per budget: the fastest device build (the build's own
"built the k-mer tables on the device in ... s" line: upload, count, passes, copy back) and the range of all, the whole
mp_idx_load wall (FASTA reading and packing on the host included), the passes, the peak the working arenas held, n_over_budget,
and the sha256 of the dumped .mpi, which must be the automatic build's for every budget.

Rows go to results/h100_idx_build.jsonl (--out), each with the device name, its power limit and what else held the device when
the genome's runs began."""
import argparse
import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import miniprot_b200 as mp  # noqa: E402
from miniprot_b200 import synth  # noqa: E402


def device():
    """name, power limit, and the memory used on it and the compute processes on it (this one's context included)"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.used,memory.total", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60)
        name, power, used, total = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        a = subprocess.run(["nvidia-smi", "--query-compute-apps=pid", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=60)
        n_apps = len([x for x in a.stdout.splitlines() if x.strip()])
        return {"device": name, "power_limit": power, "device_memory_used_at_start": used, "device_memory_total": total, "compute_processes_at_start": n_apps}
    except Exception:  # noqa: BLE001 -- a label, not a gate
        return {"device": "unknown", "power_limit": "unknown"}


def parse_size(s: str) -> int:
    m = {"k": 10, "m": 20, "g": 30}
    return int(s[:-1]) << m[s[-1].lower()] if s[-1].lower() in m else int(s)


def default_ctx():
    L = mp.lib()
    L.mpb_ctx_default.restype = C.c_void_p
    return L.mpb_ctx_default()


def build(h, g, budget, threads, mpi):
    """one mp_idx_load of FASTA `g` under `budget`: (device build s, mp_idx_load s, mem stats, .mpi sha256)"""
    L = mp.lib()
    L.mpb_ctx_set_mem_budget(h, 1)  # releases the idle arenas of the previous run
    L.mpb_ctx_set_mem_budget(h, budget)
    L.mpb_reset_stats(h)
    verbose = C.c_int32.in_dll(L, "mp_verbose")
    with tempfile.TemporaryFile() as err:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(err.fileno(), 2)
        verbose.value = 3
        try:
            t0 = time.perf_counter()
            mi = mp.idx_load(g, threads)
            t_load = time.perf_counter() - t0
        finally:
            verbose.value = 1
            os.dup2(saved, 2)
            os.close(saved)
        err.seek(0)
        text = err.read().decode(errors="replace")
    m = re.search(r"built the k-mer tables on the device in ([0-9.]+) s", text)
    if not m:
        raise RuntimeError("the index was not built on the device:\n" + text[-2000:])
    s = mp.MemStats()
    L.mpb_get_mem_stats(h, C.byref(s))
    assert L.mp_idx_dump(mpi.encode(), mi) == 0
    L.mp_idx_destroy(mi)
    with open(mpi, "rb") as f:
        digest = hashlib.file_digest(f, "sha256").hexdigest()
    os.remove(mpi)
    return float(m.group(1)), t_load, s, digest


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--configs", default="C2,C3s", help="synthetic genomes (C2, C3s, C3)")
    ap.add_argument("--budgets", default="16g,4g,1g", help="explicit budgets, after automatic mode")
    ap.add_argument("--repeat", type=int, default=3, help="runs per budget (the fastest is reported, and the range of all)")
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 8)
    ap.add_argument("--dir", default=os.environ.get("MPB_BENCH_DIR", "/tmp/mpb_bench"))
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_idx_build.jsonl"))
    a = ap.parse_args()
    h = default_ctx()
    budgets = [0] + [parse_size(x) for x in a.budgets.split(",") if x]
    rows = []
    for cfg in [x for x in a.configs.split(",") if x]:
        d = os.path.join(a.dir, cfg)
        g, _ = synth.generate(synth.CONFIGS[cfg], d)
        dev = device()
        runs = {b: [] for b in budgets}
        for _ in range(a.repeat):
            for b in budgets:
                runs[b].append(build(h, g, b, a.threads, os.path.join(d, "bench.mpi")))
        base = runs[0][0][3]
        for b in budgets:
            t_dev = [r[0] for r in runs[b]]
            best = min(runs[b], key=lambda r: r[0])
            st = best[2]
            row = {"config": cfg, "genome_bp": synth.CONFIGS[cfg].genome_len, "budget": b, "timed": "device build (upload, count, passes, copy back); load_s adds FASTA reading",
                   "build_s": round(best[0], 3), "build_s_range": [round(min(t_dev), 3), round(max(t_dev), 3)], "load_s": round(best[1], 3),
                   "n_index_passes": st.n_index_passes, "peak_held": st.peak_held, "n_over_budget": st.n_over_budget, "allowance": st.allowance,
                   "within_budget": b == 0 or st.n_over_budget > 0 or st.peak_held <= b, "mpi_sha256": best[3],
                   "identical_to_auto": all(r[3] == base for r in runs[b]), "repeat": a.repeat, **dev}
            print(json.dumps(row), flush=True)
            rows.append(row)
    mp.lib().mpb_ctx_set_mem_budget(h, 0)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "a") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    return 0 if all(r["identical_to_auto"] and r["within_budget"] for r in rows) else 1


if __name__ == "__main__":
    sys.exit(main())
