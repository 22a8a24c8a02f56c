"""Per-launch attribution of the token-row GEMMs (A_ROWS) of one forward at the bench shapes.

    python scripts/rows_probe.py [--batch 64] [--reps 20] [--skip 4,5,6] [--rows-bk 64,32] [--rounds 1]
                                 [--out FILE.json]

Records every distinct token-row GEMM launch of one forward over a batch of 512x512 planted images
(conv1, the five GEMM kinds of every coarse encoder layer on the 2D and the 3D side, the two
dual-softmax passes), adds the fine-stage GEMMs at the forward's match count (26 rows per match,
plain and with the row count read on the device), then times each one alone with CUDA events,
in child processes of their own (the engine reads its environment once per process):
  * as built;
  * with OPP_DEBUG_SKIP=4, the epilogue switched off (MMAs and loads unchanged): the difference is
    the most that hiding the epilogue behind the MMAs can give;
  * with each further OPP_DEBUG_SKIP value of --skip: 5 = no epilogue and no W loads, 6 = no
    epilogue and no A loads (the MMAs read whatever the ring holds).  A launch that gets no faster
    without its loads is not bound by them.
--rows-bk 64,32 repeats all of it once per token-row ring slot width ($OPP_ROWS_BK), the widths
alternated --rounds times (each launch keeps the median of its rounds), for an A/B in one build.
Per launch: time, issued TFLOP/s (what the tensor pipe executes: three fp16 passes over the padded
tile widths), the epilogue share, and the engine's OPP_LOG_TILES line (ring depth, accumulator
alias, cluster, N-split pair).  The card name, power limit and median SM clock are read in the same
run.  One JSON document on stdout (and in --out)."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

MARK = "rows_probe launch "

# C-ABI token-row GEMM entry points -> (batches, rows, n, k, split) from their arguments
# (include/opp_b200.h); rows of the _dyn entries are the capacity (the launch record holds the count)
SHAPES = {
    "opp_linear_act_f16": lambda a: (1, a[6], a[7], a[1] + a[3], a[10]),
    "opp_linear_act_f16_out1": lambda a: (1, a[6], a[7], a[1] + a[3], 1),
    "opp_linear_act_f16_b": lambda a: (a[7], a[8], a[9], a[1] + a[4], a[12]),
    "opp_linear_act_f16_dyn": lambda a: (1, a[6], a[9], a[1] + a[3], a[12]),
    "opp_linear_q_f16": lambda a: (a[4], a[5], a[6], a[6], a[9]),
    "opp_linear_ln": lambda a: (a[13], a[14], a[15], a[1] + a[3], a[16]),
    "opp_linear_ln_dyn": lambda a: (1, a[11], a[14], a[1] + a[3], a[15]),
    "opp_sim_lse_cols": lambda a: (a[6], a[7], a[8], a[9], a[11]),
    "opp_sim_conf_colmax": lambda a: (a[8], a[9], a[10], a[11], a[13]),
}
EPILOGUE = {"opp_linear_act_f16": "EpiStoreF16", "opp_linear_act_f16_out1": "EpiStoreF16",
            "opp_linear_act_f16_b": "EpiStoreF16", "opp_linear_act_f16_dyn": "EpiStoreF16",
            "opp_linear_q_f16": "EpiQ", "opp_linear_ln": "EpiLN", "opp_linear_ln_dyn": "EpiLN",
            "opp_sim_lse_cols": "EpiLseCol", "opp_sim_conf_colmax": "EpiConfCol"}


def _scalar(x):
    return x if isinstance(x, (int, float)) else None


def child(args):
    import torch
    import bench
    from oracle import oracle, workload
    from onepose_plus_plus_b200 import OnePosePlus_model, ops

    dev = torch.device("cuda:0")
    sd = workload.synthetic_state_dict(0)
    model = OnePosePlus_model(oracle.DEFAULT_CONFIG)
    model.load_state_dict(sd, strict=True)
    model = model.eval().to(dev)
    data, _ = workload.planted_workload(sd, bench.H, bench.W, bench.N_POINTS, bench.N_PLANTED, batch=1)
    g = torch.Generator().manual_seed(100)
    B = args.batch
    imgs = (data["query_image"] + 0.02 * torch.randn(B, 1, bench.H, bench.W, generator=g)).clamp(0, 1).to(dev)
    scale = data["query_image_scale"].expand(B, -1).contiguous().to(dev)
    bank = {k: data[k].to(dev) for k in ("keypoints3d", "descriptors3d_db", "descriptors3d_coarse_db")}

    launches, keys, keep = [], {}, []
    orig_call = ops.call
    state = {"what": None, "fine": False}

    def call_hook(name, *a):
        if name in SHAPES and state["fine"]:
            # the fine-stage launches are timed below; their tile lines are printed here, on first use
            _, _, n, k, _ = SHAPES[name](a)
            sys.stderr.write(f"{MARK}fine {n} {k}\n")
        elif name in SHAPES:
            key = (name,) + tuple(_scalar(x) for x in a) + (a[2] is not None if name == "opp_linear_act_f16_b" else None,)
            if key not in keys:
                keys[key] = len(launches)
                bt, rows, n, k, split = SHAPES[name](a)
                launches.append({"name": name, "a": a, "what": state["what"] or name, "epilogue": EPILOGUE[name],
                                 "batches": bt, "rows": rows, "n": n, "k": k, "split": int(split)})
            sys.stderr.write(f"{MARK}{keys[key]}\n")
            sys.stderr.flush()
        return orig_call(name, *a)

    # keep every tensor handed to an op alive, so the recorded device pointers stay valid
    wrapped = {}
    for fname in ("linear_act", "linear_q", "linear_ln", "sim_lse_cols", "sim_conf_colmax", "conv1_gemm"):
        fn = getattr(ops, fname)

        def w(*a, _fn=fn, _name=fname, **kw):
            keep.append((a, kw))
            prev = state["what"]
            state["what"] = state["what"] or _name
            try:
                return _fn(*a, **kw)
            finally:
                state["what"] = prev
        wrapped[fname] = fn
        setattr(ops, fname, w)
    orig_fine = model._fine

    def fine_hook(*a, **kw):
        state["fine"] = True     # timed below at the recorded match count, in both children
        try:
            return orig_fine(*a, **kw)
        finally:
            state["fine"] = False

    with torch.no_grad():
        ops.call = call_hook
        model._fine = fine_hook
        try:
            d = {"query_image": imgs, "query_image_scale": scale, **bank}
            model(d)
        finally:
            ops.call = orig_call
            for fname, fn in wrapped.items():
                setattr(ops, fname, fn)
            model._fine = orig_fine
        torch.cuda.synchronize()

        # the fine stage (model._fine, one loftr_fine layer pair) at the match count of the as-built run
        m_file = os.path.join(args.tmp, "matches.json")
        if os.environ.get("OPP_DEBUG_SKIP"):
            with open(m_file) as f:
                M = json.load(f)["M"]
        else:
            M = int(d["b_ids"].numel())
            with open(m_file, "w") as f:
                json.dump({"M": M}, f)
        rows = 26 * M
        split = model.split
        pl = 2 if split else 1
        rnd = lambda *s: (0.1 * torch.randn(*s, device=dev)).half()   # noqa: E731
        cnt = torch.tensor([M], dtype=torch.int32, device=dev)
        x, att, msg, h = rnd(rows, pl * 128), rnd(rows, pl * 128), rnd(rows, pl * 128), rnd(rows, pl * 256)
        qkv, out16 = torch.empty(rows, pl * 384, dtype=torch.float16, device=dev), torch.empty_like(x)
        out32 = torch.empty(rows, 128, dtype=torch.float32, device=dev)
        wqkv, w128, w256, w2 = rnd(384, pl * 128), rnd(128, pl * 128), rnd(256, pl * 256), rnd(128, pl * 256)
        gamma, beta = torch.ones(128, device=dev), torch.zeros(128, device=dev)
        fine = [("fine qkv 128->384 elu+1", "EpiStoreF16", 384, 128,
                 lambda **kw: ops.linear_act(x, None, wqkv, qkv, rows, 2, 256, split, **kw)),
                ("fine merge+LN 128->128", "EpiLN", 128, 128,
                 lambda **kw: ops.linear_ln(att, None, w128, False, gamma, beta, 1, rows, split, out16=out16, **kw)),
                ("fine mlp0 256->256 relu", "EpiStoreF16", 256, 256,
                 lambda **kw: ops.linear_act(x, msg, w256, h, rows, 1, 256, split, **kw)),
                ("fine mlp2+LN 256->128 +resid fp32", "EpiLN", 128, 256,
                 lambda **kw: ops.linear_ln(h, None, w2, False, gamma, beta, 1, rows, split, resid=x, out32=out32,
                                            **kw))]
        if M:
            for what, epi, n, k, fn in fine:
                for dyn in (False, True):
                    kw = {"count": cnt, "rows_per_count": 26} if dyn else {}
                    name = ("opp_linear_ln" if epi == "EpiLN" else "opp_linear_act_f16") + ("_dyn" if dyn else "")
                    launches.append({"name": name, "fn": (lambda fn=fn, kw=kw: fn(**kw)),
                                     "what": what + (" dyn" if dyn else ""), "epilogue": epi, "batches": 1,
                                     "rows": rows, "n": n, "k": k, "split": int(split)})
                    sys.stderr.write(f"{MARK}{len(launches) - 1}\n")
                    sys.stderr.flush()
                    launches[-1]["fn"]()
        torch.cuda.synchronize()

        sampler = bench.ClockSampler(0)
        t0 = time.time()
        res = []
        for i, L in enumerate(launches):
            fn = L["fn"] if "fn" in L else (lambda L=L: orig_call(L["name"], *L["a"]))
            ms = bench.cuda_time(fn, args.reps, warm=3)
            res.append({k: v for k, v in L.items() if k not in ("fn", "a")} | {"ms": ms, "index": i})
        clocks = sampler.stop(t0, time.time())
    print(json.dumps({"launches": res, "clocks": clocks, "matches": M}))


def run_child(args, tmp, env_extra):
    env = dict(os.environ, OPP_LOG_TILES="1", **env_extra)
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--batch", str(args.batch),
                        "--reps", str(args.reps), "--tmp", tmp], env=env, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stderr[-4000:])
        raise SystemExit(f"child ({env_extra}) failed with exit code {p.returncode}")
    out = json.loads(p.stdout.strip().splitlines()[-1])
    # tile lines of the token-row mode (0 = A_ROWS), attributed to the launch they follow
    tiles, cur = {}, None
    for line in p.stderr.splitlines():
        if line.startswith(MARK):
            cur = line[len(MARK):]
            cur = int(cur) if cur.isdigit() else cur
        elif line.startswith("opp gemm tile: mode 0"):
            if cur is not None:
                tiles.setdefault(cur, []).append(line[len("opp gemm tile: "):])
    # a launch without a line of its own shares the tile configuration of an earlier one
    # (the log key has no epilogue: the second dual-softmax pass shares the line of the first)
    for i, L in enumerate(out["launches"]):
        L["tile"] = tiles.get(f"fine {L['n']} {L['k']}") if L["what"].startswith("fine") else tiles.get(i)
        if L["tile"] is None:
            shape = lambda P: (P["n"], P["k"], P["split"], P["batches"])   # noqa: E731
            same = [P["tile"] for P in out["launches"][:i] if P["tile"] and shape(P) == shape(L)]
            same.sort(key=lambda t: 0 if t in [P["tile"] for P in out["launches"][:i]
                                                if P["epilogue"] == L["epilogue"]] else 1)
            L["tile"] = same[0] if same else None
    return out


def tile_field(tile, name):
    f = tile.split()
    return int(f[f.index(name) + 1])


def device_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        info["power_limit"], info["sm_max_clock"] = [x.strip() for x in q.stdout.strip().split(",")][:2]
    except (OSError, ValueError, subprocess.SubprocessError):
        info["power_limit"] = None
    return info


def launch_key(L):
    return (L["what"], L["name"], L["batches"], L["rows"], L["n"], L["k"])


def table(full, arms):
    """per-launch rows of the as-built child `full`, with the time of each OPP_DEBUG_SKIP arm"""
    skip_ms = {v: {launch_key(S): S["ms"] for S in a["launches"]} for v, a in arms.items()}
    rows = []
    for L in full["launches"]:
        r = {k: L[k] for k in ("what", "name", "epilogue", "batches", "rows", "n", "k", "ms", "tile")}
        r["ms_skip"] = {v: m.get(launch_key(L)) for v, m in skip_ms.items()}
        off = r["ms_skip"].get("4")
        r["ms_epilogue_off"] = off
        r["epilogue_share"] = None if off is None else 1.0 - off / L["ms"]
        if L["tile"]:
            t = L["tile"][0]
            n_tiles = math.ceil(tile_field(t, "n") / tile_field(t, "block_n"))
            tiles = L["batches"] * math.ceil(L["rows"] / 128) * n_tiles
            issued = (3 if L["split"] else 1) * 2.0 * tiles * 128 * tile_field(t, "mma_n") * tile_field(t, "k")
            r["issued_tflop"] = issued / 1e12
            r["issued_tflops"] = issued / (L["ms"] * 1e-3) / 1e12
        rows.append(r)
    return rows


def median_of(runs):
    """one child result whose launch times are the medians over `runs` (same launches, same order)"""
    out = dict(runs[0])
    out["launches"] = [dict(L, ms=statistics.median(R["launches"][i]["ms"] for R in runs))
                       for i, L in enumerate(runs[0]["launches"])]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--skip", default="4", help="comma-separated OPP_DEBUG_SKIP arms (4 = no epilogue, "
                                                 "5 = + no W loads, 6 = + no A loads)")
    ap.add_argument("--rows-bk", default="", help="comma-separated OPP_ROWS_BK arms (default: as built)")
    ap.add_argument("--rounds", type=int, default=1, help="alternations of the --rows-bk arms")
    ap.add_argument("--out")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tmp", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rows_probe needs a CUDA device")
    skips = [v for v in args.skip.split(",") if v]
    bks = [v for v in args.rows_bk.split(",") if v] or [None]
    fulls = {bk: [] for bk in bks}
    arms = {bk: {v: [] for v in skips} for bk in bks}
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.rounds):
            for bk in bks:
                env = {"OPP_ROWS_BK": bk} if bk else {}
                fulls[bk].append(run_child(args, tmp, env))
                for v in skips:
                    arms[bk][v].append(run_child(args, tmp, env | {"OPP_DEBUG_SKIP": v}))
    doc = {"device": device_info() | {"sms": torch.cuda.get_device_properties(0).multi_processor_count},
           "batch": args.batch, "reps": args.reps, "rounds": args.rounds, "skip_arms": skips,
           "note": "issued = (3 if split) fp16 MMA passes x 128 rows x mma_n columns x K per tile; rows of the "
                   "dyn launches = the capacity = the count; ms_skip[v] = the same launch with OPP_DEBUG_SKIP=v "
                   "in another process (4: no epilogue, 5: + no W loads, 6: + no A loads); ms = median over "
                   "the rounds", "arms": {}}
    for bk in bks:
        full = median_of(fulls[bk])
        rows = table(full, {v: median_of(a) for v, a in arms[bk].items()})
        doc["arms"][bk or "as built"] = {"clocks": full["clocks"], "matches": full["matches"], "launches": rows}
        sys.stderr.write(f"== OPP_ROWS_BK={bk or '(as built)'}\n")
        for r in rows:
            sk = "  ".join(f"skip{v} {r['ms_skip'][v] if r['ms_skip'][v] is not None else float('nan'):7.3f}"
                           for v in skips)
            sys.stderr.write(f"{r['what'][:34]:<34} {r['name'][4:]:<20} {r['ms']:7.3f} ms  {sk}  "
                             f"{r.get('issued_tflops', 0):6.1f} TF  {(r['tile'] or ['?'])[0]}\n")
    s = json.dumps(doc)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
