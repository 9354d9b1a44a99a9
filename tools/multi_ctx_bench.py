"""Time mpb_map_file_multi end to end on the C2 synthetic workload: one context, two contexts on one GPU ("0,0": a second mini-batch
in flight), and one context per visible GPU when there are several.

    python tools/multi_ctx_bench.py [--workload C2] [--repeats 3] [--configs 0 0,0 ...] [--out result.jsonl]

For each setting: proteins/s over the whole query file (reading, mapping, formatting and writing the PAF; the index is resident
beforehand), and per context the wall-clock split of the dispatcher's phases (mpb_stats_t.ms_wall: S1, H1, S2, H2, S3, H3).  The
PAF of every setting must equal the one-context PAF byte for byte.  Inputs and outputs go to a temporary directory.
"""
import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import miniprot_b200 as mp  # noqa: E402
from miniprot_b200 import synth  # noqa: E402

PHASES = ("S1", "H1", "S2", "H2", "S3", "H3")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C2", choices=sorted(synth.CONFIGS))
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--configs", nargs="*", help="device lists such as 0 or 0,0 (default: 0, 0,0 and every visible device)")
    ap.add_argument("--out", help="also append the result lines to this file")
    a = ap.parse_args()

    import torch

    n_dev = torch.cuda.device_count()
    configs = a.configs or (["0", "0,0"] + ([",".join(str(i) for i in range(n_dev))] if n_dev > 1 else []))
    spec = synth.CONFIGS[a.workload]
    lines = []
    with tempfile.TemporaryDirectory() as d:
        g, _ = synth.generate(spec, d)
        prot = synth.shard_queries(spec, d, 0)
        n_prot = sum(1 for line in open(prot) if line.startswith(">"))
        n_res = sum(len(line.strip()) for line in open(prot) if not line.startswith(">"))
        # the whole file is one mini-batch, as in a bench.py step: one context maps it in one piece, n contexts in n units
        mo = mp.mapopt(mini_batch_size=n_res)
        t0 = time.time()
        mi = mp.idx_load(g, os.cpu_count() or 8)
        t_idx = time.time() - t0
        want = None
        for cfg in configs:
            devs = [int(x) for x in cfg.split(",")]
            ctxs = [mp.Context(x) for x in devs]
            out = os.path.join(d, "o.paf")
            mp.map_file_multi(ctxs, mi, prot, out, mo)  # warm-up: index resident in every context, arenas grown
            for c in ctxs:
                c.reset_stats()
            wall = []
            for _ in range(a.repeats):
                t0 = time.time()
                mp.map_file_multi(ctxs, mi, prot, out, mo)
                wall.append(time.time() - t0)
            digest = hashlib.sha256(open(out, "rb").read()).hexdigest()
            want = want or digest
            per_ctx = []
            for dev, c in zip(devs, ctxs):
                s = c.stats()
                per_ctx.append({"device": dev, "ms_wall_per_run": {p: round(s.ms_wall[k] / a.repeats, 1) for k, p in enumerate(PHASES)},
                                "dp_cells_per_run": (s.dp_cells_ext + s.dp_cells_tb) // a.repeats})
            for c in ctxs:
                c.close()
            best = min(wall)
            line = {"tool": "multi_ctx_bench", "workload": a.workload, "devices": cfg, "n_ctx": len(devs), "proteins": n_prot, "mini_batch_size": n_res, "repeats": a.repeats,
                    "s_per_run": [round(w, 3) for w in wall], "proteins_per_s": round(n_prot / best, 1), "paf_sha256": digest[:16],
                    "paf_same_as_one_context": digest == want, "per_ctx": per_ctx, "index_load_s": round(t_idx, 2),
                    "gpu": torch.cuda.get_device_name(devs[0])}
            print(json.dumps(line), flush=True)
            lines.append(line)
        mp.lib().mp_idx_destroy(mi)
    if a.out:
        with open(a.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    if not all(line["paf_same_as_one_context"] for line in lines):
        sys.exit("PAF differs from the one-context PAF")


if __name__ == "__main__":
    main()
