"""Per-launch attribution of the implicit-GEMM convolutions of one forward at the bench shapes.

    python scripts/conv_probe.py [--batch 64] [--reps 20] [--out FILE.json]

Records every distinct `opp_conv2d_nhwc` / `opp_conv_win` launch of one forward over a batch of
512x512 planted images (plus the window head of bench.py's fine_head block), then times each one
alone with CUDA events, twice, each in a child process of its own (the engine reads its
environment once per process):
  * as built;
  * with OPP_DEBUG_SKIP=4, the epilogue switched off (MMAs and loads unchanged): the difference is
    the most that hiding the epilogue behind the MMAs can give.
Per launch: time, algorithmic and issued TFLOP/s (issued = what the tensor pipe executes: three
fp16 passes over the padded tile widths), tiles per SM, and the engine's OPP_LOG_TILES line (ring
depth, accumulator alias, cluster).  The card name, power limit and median SM clock are read in
the same run.  One JSON document on stdout (and in --out)."""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MARK = "conv_probe launch "


def true_channels(c_pad):
    return 196 if c_pad == 208 else c_pad     # the only padded width of this backbone


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

    launches, keys = [], {}
    orig_conv, orig_win = ops.conv2d_nhwc, ops.conv_win

    def record(kind, fn, key, desc, a, kw):
        if key not in keys:
            keys[key] = len(launches)
            launches.append({"kind": kind, "fn": fn, "a": a, "kw": kw, **desc})
        sys.stderr.write(f"{MARK}{keys[key]}\n")
        sys.stderr.flush()

    def conv_hook(x, w, bias, out, ksize, stride, split, act=0, resid=None, slope=0.01, tok=None, pe=None,
                  up=None):
        Bn, h, wd, _ = x.shape
        oh, ow = (h - 1) // stride + 1, (wd - 1) // stride + 1
        cin, cout = w.shape[1] // (ksize * ksize * (2 if split else 1)), w.shape[0]
        key = ("conv", tuple(x.shape), tuple(w.shape), ksize, stride, act, resid is not None, tok is not None,
               up is not None)
        what = f"{ksize}x{ksize}{'/2' if stride == 2 else ''} {cin}->{cout} @{oh}x{ow}"
        what += "".join(s for s, on in ((" +resid", resid is not None), (" +tok", tok is not None),
                                        (" +up2x", up is not None)) if on)
        desc = {"what": what, "epilogue": "EpiConvUp" if up is not None else "EpiConv",
                "m_tiles": Bn * math.ceil(oh / 8) * math.ceil(ow / 16), "rows_per_tile": 128,
                "pixels": Bn * oh * ow, "cin": cin, "cout": cout, "taps": ksize * ksize}
        a = (x, w, bias, out, ksize, stride, split)
        kw = dict(act=act, resid=resid, slope=slope, tok=tok, pe=pe, up=up)
        record("conv", orig_conv, key, desc, a, kw)
        return orig_conv(*a, **kw)

    def win_hook(x, w, bias, out, win, split, m, act=0, slope=0.01, b_ids=None, j_ids=None, wc=0, stride=4,
                 org=0, count=None):
        cin, cout = w.shape[1] // (9 * (2 if split else 1)), w.shape[0]
        key = ("win", tuple(x.shape), tuple(w.shape), win, m, j_ids is not None)
        per_tile = 128 // (ops.conv_win_pitch(win) * win)
        desc = {"what": f"window 3x3 {cin}->{cout} {win}x{win} x {m} matches ({'A' if j_ids is not None else 'B'})",
                "epilogue": "EpiWin", "m_tiles": math.ceil(m / per_tile),
                "rows_per_tile": per_tile * ops.conv_win_pitch(win) * win,
                "pixels": m * win * win, "cin": cin, "cout": cout, "taps": 9}
        a = (x, w, bias, out, win, split, m)
        kw = dict(act=act, slope=slope, b_ids=b_ids, j_ids=j_ids, wc=wc, stride=stride, org=org, count=count)
        record("win", orig_win, key, desc, a, kw)
        return orig_win(*a, **kw)

    with torch.no_grad():
        ops.conv2d_nhwc, ops.conv_win = conv_hook, win_hook
        try:
            d = {"query_image": imgs, "query_image_scale": scale, **bank}
            model(d)
            # the window head as bench.py's fine_head block runs it (the forward may take the dense one).
            # Without epilogues the forward finds no matches: that child takes the first child's list.
            ids_file = os.path.join(args.tmp, "match_ids.pt")
            if os.environ.get("OPP_DEBUG_SKIP"):
                b_ids, j_ids = (t.to(dev) for t in torch.load(ids_file))
            else:
                b_ids, j_ids = d["b_ids"], d["j_ids"]
                torch.save((b_ids.cpu(), j_ids.cpu()), ids_file)
            x1_lat = model._backbone(imgs, defer_fine=True)[1]
            M = int(b_ids.numel())
            if M:
                model._fine_head_windows(x1_lat, b_ids, j_ids, M, bench.W // 8, 4)
        finally:
            ops.conv2d_nhwc, ops.conv_win = orig_conv, orig_win
        torch.cuda.synchronize()

        sampler = bench.ClockSampler(0)
        t0 = time.time()
        res = []
        for L in launches:
            ms = bench.cuda_time(lambda: L["fn"](*L["a"], **L["kw"]), args.reps, warm=3)
            res.append({k: v for k, v in L.items() if k not in ("fn", "a", "kw")} | {"ms": ms})
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
    # tile lines of the conv modes (1 = A_CONV, 2 = A_WIN), attributed to the launch they follow
    tiles, cur = {}, None
    for line in p.stderr.splitlines():
        if line.startswith(MARK):
            cur = int(line[len(MARK):])
        elif line.startswith("opp gemm tile: mode 1") or line.startswith("opp gemm tile: mode 2"):
            if cur is not None:
                tiles.setdefault(cur, []).append(line[len("opp gemm tile: "):])
    # a launch without a line of its own shares the tile configuration of an earlier one
    for i, L in enumerate(out["launches"]):
        L["tile"] = tiles.get(i)
        if L["tile"] is None:
            same = [P["tile"] for P in out["launches"][:i] if P["tile"] and P["epilogue"] == L["epilogue"]
                    and (P["cin"], P["cout"], P["taps"]) == (L["cin"], L["cout"], L["taps"])]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tmp", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("conv_probe needs a CUDA device")
    with tempfile.TemporaryDirectory() as tmp:
        full = run_child(args, tmp, {})
        noepi = run_child(args, tmp, {"OPP_DEBUG_SKIP": "4"})
    skip_ms = {S["what"]: S["ms"] for S in noepi["launches"]}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = []
    for L in full["launches"]:
        S = {"ms": skip_ms[L["what"]]}
        alg = 2.0 * L["pixels"] * true_channels(L["cin"]) * true_channels(L["cout"]) * L["taps"]
        r = {k: L[k] for k in ("what", "epilogue", "ms", "tile")} | {"ms_epilogue_off": S["ms"]}
        r["epilogue_share"] = 1.0 - S["ms"] / L["ms"]
        r["algorithmic_tflops"] = alg / (L["ms"] * 1e-3) / 1e12
        if L["tile"]:
            t = L["tile"][0]
            n_tiles = math.ceil(tile_field(t, "n") / tile_field(t, "block_n"))
            conv_c = tile_field(t, "conv_c")
            k_issued = L["taps"] * (conv_c if conv_c % 64 == 16 else math.ceil(conv_c / 64) * 64)
            tiles = L["m_tiles"] * n_tiles
            issued = 3 * 2.0 * tiles * 128 * tile_field(t, "mma_n") * k_issued
            r["issued_tflops"] = issued / (L["ms"] * 1e-3) / 1e12
            r["tiles_per_sm"] = tiles / sms
            r["us_per_tile"] = L["ms"] * 1e3 / math.ceil(tiles / sms)
        rows.append(r)
    doc = {"device": device_info() | {"sms": sms}, "batch": args.batch, "reps": args.reps,
           "clocks": full["clocks"], "clocks_epilogue_off": noepi["clocks"], "matches": full["matches"],
           "launches": rows,
           "note": "issued = 3 fp16 MMA passes x 128 rows x mma_n columns x K actually issued per tile; "
                   "ms_epilogue_off = the same launch with OPP_DEBUG_SKIP=4 (no epilogue) in another process"}
    for r in rows:
        sys.stderr.write(f"{r['what']:<44} {r['ms']:8.3f} ms  no-epi {r['ms_epilogue_off']:8.3f} ms "
                         f"({100 * r['epilogue_share']:5.1f} %)  {r.get('issued_tflops', 0):6.1f} TF issued  "
                         f"{(r['tile'] or ['?'])[0]}\n")
    s = json.dumps(doc)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
