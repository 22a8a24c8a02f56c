"""A/B of the engine's K chunk width (OPP_CONV_BK) — or of any other engine switch — per launch.

    python scripts/chunk_probe.py [--batch 64] [--reps 20] [--rounds 2] [--rows]
                                  [--config NAME=VAR=VAL[,VAR=VAL...]]... [--out FILE.json]

Runs the child of scripts/conv_probe.py (every distinct conv launch of one forward at the bench
shapes, plus the window head), and with --rows also the child of scripts/rows_probe.py (the
token-row GEMMs), once per configuration and round, configurations alternating within a round.  The
engine reads its environment once per process, so every configuration runs in a process of its own.
Default configurations: bk64 (OPP_CONV_BK=64) and bk32 (OPP_CONV_BK=32).  A configuration with
OPP_DEBUG_SKIP (W or A loads skipped: timing only) is run after a plain one, whose match list it
reuses.

Per launch and configuration: the median time over the rounds, the ring depth ("stages") and K
chunk width ("bk") of the engine's OPP_LOG_TILES line, and the ratio to the first configuration.
The card name, power limit and the median SM clock of every child are read in the same run.  One
JSON document on stdout (and in --out); a table on stderr."""
import argparse
import json
import os
import re
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import conv_probe  # noqa: E402
import rows_probe  # noqa: E402


def parse_config(text):
    name, _, env = text.partition("=")
    pairs = [p.split("=", 1) for p in env.split(",") if p]
    if not name or any(len(p) != 2 for p in pairs):
        raise SystemExit(f"bad --config {text!r}: want NAME=VAR=VAL[,VAR=VAL...]")
    return name, dict(pairs)


def tile_info(tile):
    if not tile:
        return {"stages": None, "bk": None}
    f = tile[0].split()
    return {k: int(f[f.index(k) + 1]) if k in f else None for k in ("stages", "bk")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rows", action="store_true", help="also the token-row GEMMs (rows_probe)")
    ap.add_argument("--config", action="append", default=[])
    ap.add_argument("--out")
    args = ap.parse_args()
    configs = [parse_config(c) for c in args.config] or [("bk64", {"OPP_CONV_BK": "64"}),
                                                         ("bk32", {"OPP_CONV_BK": "32"})]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("chunk_probe needs a CUDA device")
    probes = [("conv", conv_probe)] + ([("rows", rows_probe)] if args.rows else [])
    # per (probe, config): list over rounds of {launch what: (ms, tile)}, and the clocks of each child
    times, clocks, tiles = {}, {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for pname, mod in probes:
            ptmp = os.path.join(tmp, pname)
            os.makedirs(ptmp)
            if any("OPP_DEBUG_SKIP" in env for _, env in configs) and "OPP_DEBUG_SKIP" in configs[0][1]:
                mod.run_child(args, ptmp, {})   # writes the match list the skip children read
            for _ in range(args.rounds):
                for cname, env in configs:
                    out = mod.run_child(args, ptmp, env)
                    clocks.setdefault((pname, cname), []).append(out["clocks"])
                    for L in out["launches"]:
                        # the window launches' names carry the match count, which may differ by a few
                        # between configurations that round differently
                        what = re.sub(r" x \d+ matches", " x M matches", L["what"])
                        key = (pname, what + (f" [{L['name']}]" if pname == "rows" else ""))
                        times.setdefault(key, {}).setdefault(cname, []).append(L["ms"])
                        tiles.setdefault(key, {})[cname] = tile_info(L["tile"])
    base = configs[0][0]
    rows = []
    for (pname, what), per in times.items():
        r = {"probe": pname, "what": what}
        for cname, _ in configs:
            if cname not in per:
                continue
            ms = statistics.median(per[cname])
            r[cname] = {"ms": ms, "ms_rounds": per[cname], **tiles[(pname, what)][cname]}
            if base in per:
                r[cname]["vs_" + base] = ms / statistics.median(per[base])
        rows.append(r)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    doc = {"device": conv_probe.device_info() | {"sms": sms}, "batch": args.batch, "reps": args.reps,
           "rounds": args.rounds, "configs": {c: e for c, e in configs},
           "clocks": {f"{p} {c}": v for (p, c), v in clocks.items()}, "launches": rows}
    head = "".join(f" {c:>26}" for c, _ in configs)
    sys.stderr.write(f"{doc['device']}\n{'launch':<58}{head}\n")
    for r in rows:
        cells = ""
        for c, _ in configs:
            v = r.get(c)
            cells += (f" {v['ms']:8.3f} ms x{v.get('vs_' + base, 1):5.3f} s{v['stages']} k{v['bk']}" if v
                      else f" {'-':>26}")
        sys.stderr.write(f"{r['what'][:58]:<58}{cells}\n")
    for (p, c), v in clocks.items():
        sys.stderr.write(f"clock {p} {c}: {[x.get('sm_mhz') for x in v]} MHz\n")
    s = json.dumps(doc)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
