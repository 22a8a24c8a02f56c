"""pytest -m gpu: several objects in one forward (model.set_banks + data["object_ids"]).

* every frame of a B = 8 batch over three objects (N = 1237, 5000, 300: none a multiple of 32, and
  the 300-point object's padding covers whole 32-row groups) equals the one-object call of its
  object (set_bank + a one-frame forward), in both precisions and at B = 1, with the padded bank
  state filled with large-norm garbage;
* permuting frames and object ids together permutes the outputs;
* conf_matrix ("eager" and lazy .materialize()): padded rows exactly 0, valid rows those of the
  one-object matrix;
* one CUDA graph replayed with two assignments equals the eager forward of each;
* an object with no match in its frame, and a set whose frames all show one object;
* a two-object PoseTracker against the crops, matches and poses of one-object calls;
* the kernels' new arguments against numpy over the valid rows only (row_count in the lse / conf
  passes, bank_of_batch in the match selection and the fine gather), with padded rows crafted to
  win every column maximum and dominate every column lse if they were read."""
import numpy as np
import pytest
import torch

from onepose_plus_plus_b200 import ops, pnp, tracking
from oracle import workload
from tests import parity

pytestmark = pytest.mark.gpu

H, W = 256, 320
NS = (1237, 5000, 300)
OIDS = [2, 0, 0, 1, 2, 1, 0, 2]


@pytest.fixture(scope="module")
def objects():
    """Three planted objects (own image, own bank) and 8 frames: each frame is its object's image
    plus fresh noise."""
    sd = workload.synthetic_state_dict(0)
    objs = []
    for k, n in enumerate(NS):
        d, _ = workload.planted_workload(sd, H, W, n_points=n, n_planted=min(700, n // 2), batch=1, seed=3 + 7 * k,
                                         with_scale=False)
        d["keypoints3d"] = d["keypoints3d"] * (1.0 + 0.5 * k) + 0.3 * k     # different extents and offsets
        objs.append(d)
    g = torch.Generator().manual_seed(4)
    frames = torch.cat([(objs[o]["query_image"] + 0.01 * torch.randn(1, 1, H, W, generator=g)).clamp(0, 1)
                        for o in OIDS], 0)
    scale = 0.7 + 0.8 * torch.rand(len(OIDS), 2, generator=g)
    return objs, frames, scale


def _banks(objs):
    return [(o["keypoints3d"].cuda(), o["descriptors3d_db"].cuda(), o["descriptors3d_coarse_db"].cuda())
            for o in objs]


def _garbage(m, seed=0):
    """Fill the padding of the resident set's state with large-norm finite values."""
    m._ensure_plan(torch.device("cuda"))
    st = m._resident_set_state()
    g = torch.Generator(device="cuda").manual_seed(seed)
    for k, n in enumerate(st["n_rows"].tolist()):
        rest = st["N"] - n
        if rest == 0:
            continue
        st["d3_l0"][k, n:] = (60 * torch.randn(rest, st["d3_l0"].shape[2], device="cuda", generator=g)).half()
        st["kpts"][k, n:] = 1e3 * torch.randn(rest, 3, device="cuda", generator=g)
        st["fine"][k, :, n:] = 1e3 * torch.randn(st["fine"].shape[1], rest, device="cuda", generator=g)


def _set_forward(m, frames, scale, oids):
    d = {"query_image": frames.cuda(), "query_image_scale": scale.cuda(),
         "object_ids": torch.tensor(oids, dtype=torch.int32)}
    m(d)
    torch.cuda.synchronize()
    return d


def _one_object(m, objs, frames, scale, b, o):
    m.set_bank(*_banks(objs)[o])
    d = {"query_image": frames[b:b + 1].cuda(), "query_image_scale": scale[b:b + 1].cuda()}
    m(d)
    torch.cuda.synchronize()
    return {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in d.items()}


def _refs(m, objs, frames, scale, oids):
    refs = [_one_object(m, objs, frames, scale, b, o) for b, o in enumerate(oids)]
    m.clear_bank()
    return refs


def _check_frames(got, refs, precision="fp16x3"):
    reps = []
    for b, ref in enumerate(refs):
        g = parity.select_image(got, b)
        if ref["b_ids"].numel() == 0:
            assert g["b_ids"].numel() == 0, b
            reps.append({"M": 0})
        elif precision == "fp16x3":
            reps.append(parity.compare(g, ref, max_borderline=0))
        else:
            reps.append(_compare_fp16(g, ref))
    return reps


def _compare_fp16(got, ref):
    """Single fp16 operands move mconf by up to ~1e-2 when only the order of the coarse KV sums
    changes (the one-object path alone does, between a frame run alone and inside a batch: DESIGN
    §7 f5), and the set sums at N_max instead of N_k: the same matches up to a few near the
    threshold, mconf within 2e-2, mkpts_3d_db exact on the common ones."""
    g = list(zip(got["i_ids"].tolist(), got["j_ids"].tolist()))
    r = list(zip(ref["i_ids"].tolist(), ref["j_ids"].tolist()))
    common = set(g) & set(r)
    assert len(common) >= 0.95 * max(len(r), len(g)), (len(common), len(g), len(r))
    for t in set(g) ^ set(r):
        c = (got["mconf"][g.index(t)] if t in g else ref["mconf"][r.index(t)]).item()
        assert abs(c - parity.THR) <= 2e-2, (t, c)
    gi = torch.tensor([g.index(t) for t in r if t in common], dtype=torch.long)
    ri = torch.tensor([i for i, t in enumerate(r) if t in common], dtype=torch.long)
    assert (got["mconf"].cpu()[gi] - ref["mconf"][ri]).abs().max().item() <= 2e-2
    assert torch.equal(got["mkpts_3d_db"].cpu()[gi], ref["mkpts_3d_db"][ri])
    return {"M": len(r)}


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_each_frame_equals_its_one_object_call(objects, precision):
    objs, frames, scale = objects
    m = parity.cuda_model(0, precision)
    refs = _refs(m, objs, frames, scale, OIDS)
    assert sum(r["b_ids"].numel() for r in refs) > 8 * 50
    m.set_banks(_banks(objs))
    _garbage(m)
    try:
        got = _set_forward(m, frames, scale, OIDS)
        reps = _check_frames(got, refs, precision)
        print(precision, [r["M"] for r in reps])
        # B = 1, object_ids on the device
        one = {"query_image": frames[3:4].cuda(), "query_image_scale": scale[3:4].cuda(),
               "object_ids": torch.tensor([1], device="cuda")}
        m(one)
        _check_frames(one, refs[3:4], precision)
    finally:
        m.clear_bank()


def test_layer_norm_eps_does_not_hide_a_scale(objects, monkeypatch):
    """LayerNorm follows every attention message, so a message scaled by a constant factor only
    shows through the LayerNorm eps.  With eps raised to 0.1 in every LayerNorm GEMM, a frame whose
    cached layer-1 state were divided by N_k while the forward's query multiplies by N_max would
    move; with the matching v_len it still equals its one-object call."""
    real = ops.linear_ln

    def linear_ln(*a, **k):
        k["eps"] = 0.1
        return real(*a, **k)
    monkeypatch.setattr(ops, "linear_ln", linear_ln)
    objs, frames, scale = objects
    m = parity.cuda_model(0)
    refs = _refs(m, objs, frames, scale, OIDS)
    assert sum(r["b_ids"].numel() for r in refs) > 8 * 20
    m.set_banks(_banks(objs))
    _garbage(m)
    try:
        _check_frames(_set_forward(m, frames, scale, OIDS), refs)
    finally:
        m.clear_bank()


def test_permuting_frames_permutes_outputs(objects):
    objs, frames, scale = objects
    m = parity.cuda_model(0)
    m.set_banks(_banks(objs))
    _garbage(m)
    try:
        got = _set_forward(m, frames, scale, OIDS)
        perm = [5, 2, 7, 0, 3, 6, 1, 4]
        gp = _set_forward(m, frames[perm], scale[perm], [OIDS[p] for p in perm])
        for nb, p in enumerate(perm):
            a, b = parity.select_image(gp, nb), parity.select_image(got, p)
            for k in ("i_ids", "j_ids", "mkpts_3d_db"):
                assert torch.equal(a[k], b[k]), (nb, k)
            for k in ("mconf", "mkpts_query_f", "expec_f"):
                assert torch.allclose(a[k], b[k], rtol=0, atol=1e-5), (nb, k)
    finally:
        m.clear_bank()


def test_conf_matrix_padded_rows_are_zero(objects):
    objs, frames, scale = objects
    m = parity.cuda_model(0)
    S = (H // 8) * (W // 8)
    refs = []
    for b, o in enumerate(OIDS):
        m.set_bank(*_banks(objs)[o])
        d = {"query_image": frames[b:b + 1].cuda(), "query_image_scale": scale[b:b + 1].cuda()}
        m(d)
        refs.append(d["conf_matrix"][0].clone())
    m.set_banks(_banks(objs))
    _garbage(m)
    try:
        for mode in ("eager", "lazy"):
            m.conf_matrix_mode = mode
            d = _set_forward(m, frames, scale, OIDS)
            conf = d["conf_matrix"] if mode == "eager" else d["conf_matrix"].materialize()
            assert conf.shape == (8, max(NS), S)
            for b, o in enumerate(OIDS):
                n = NS[o]
                assert (conf[b, n:] == 0).all().item(), (mode, b)
                # the KV state sums run at N_max instead of N: rounding only (measured 1.4e-5)
                assert (conf[b, :n] - refs[b]).abs().max().item() <= 5e-5, (mode, b)
    finally:
        m.conf_matrix_mode = "eager"
        m.clear_bank()


def test_one_graph_serves_every_assignment(objects):
    objs, frames, scale = objects
    m = parity.cuda_model(0)
    m.set_banks(_banks(objs))
    _garbage(m)
    m.conf_matrix_mode = "lazy"
    keys = ("b_ids", "i_ids", "j_ids", "mconf", "mkpts_3d_db", "mkpts_query_f", "expec_f")
    try:
        other = [1, 1, 0, 2, 0, 2, 1, 0]
        eager = [_set_forward(m, frames, scale, oids) for oids in (OIDS, other)]
        eager = [{k: d[k].clone() for k in keys} for d in eager]
        m.enable_cuda_graphs(True)
        graph = None
        for i in (0, 1, 0):
            d = {"query_image": frames.cuda(), "query_image_scale": scale.cuda(),
                 "object_ids": torch.tensor((OIDS, other)[i], device="cuda")}
            m(d)
            assert len(m._graphs) == 1
            g = next(iter(m._graphs.values()))["graph"]
            assert graph is None or g is graph      # captured once, replayed for every assignment
            graph = g
            for k in keys:
                assert torch.equal(d[k], eager[i][k]), (i, k)
    finally:
        m.enable_cuda_graphs(False)
        m.conf_matrix_mode = "eager"
        m.clear_bank()


def test_degenerate_assignments(objects):
    objs, frames, scale = objects
    m = parity.cuda_model(0)
    # a fourth object with an unplanted (random) bank, and frame 1 a random image assigned to it:
    # no match in that frame, as in its one-object call
    rnd = workload.random_workload(H, W, n_points=800, batch=1, seed=7)
    objs = objs + [{k: rnd[k] for k in ("keypoints3d", "descriptors3d_db", "descriptors3d_coarse_db")}]
    oids = list(OIDS)
    oids[1] = 3
    fr = frames.clone()
    fr[1] = rnd["query_image"][0]
    refs = _refs(m, objs, fr, scale, oids)
    assert refs[1]["b_ids"].numel() == 0
    m.set_banks(_banks(objs))
    _garbage(m)
    try:
        got = _set_forward(m, fr, scale, oids)
        assert (got["b_ids"] == 1).sum().item() == 0
        _check_frames(got, refs)
        # every frame on object 1: the whole batch equals set_bank of object 1
        got = _set_forward(m, frames, scale, [1] * 8)
    finally:
        m.clear_bank()
    m.set_bank(*_banks(objs)[1])
    ref = {"query_image": frames.cuda(), "query_image_scale": scale.cuda()}
    m(ref)
    m.clear_bank()
    parity.compare(got, {k: v.cpu() for k, v in ref.items() if torch.is_tensor(v)}, max_borderline=0)


# ------------------------------------------------------------------------------------------------
# PoseTracker with two objects
# ------------------------------------------------------------------------------------------------
def test_pose_tracker_two_objects():
    from tests import test_tracking_gpu as ttg
    sd = workload.synthetic_state_dict(0)
    m = parity.cuda_model(0)
    scenes = [ttg._tracking_scene(sd, n_points=n, seed=s) for n, s in ((2000, 1), (1700, 5))]
    banks = [tuple(t.cuda() for t in bank) for _, bank, _ in scenes]
    corners = np.stack([c for _, _, c in scenes])
    K = ttg._cameras()
    rng = np.random.default_rng(3)
    Hf, Wf = ttg.FRAME_HW
    frames = []
    for t in range(5):    # camera b shows object b
        fr = []
        for b, (ox, oy) in enumerate(ttg.OFFSETS):
            f = ttg._frame(rng, Hf, Wf).astype(np.int16)
            f[oy:oy + ttg.CROP, ox:ox + ttg.CROP] = scenes[b][0]
            f += rng.integers(-3, 4, f.shape).astype(np.int16)
            fr.append(np.clip(f, 0, 255).astype(np.uint8))
        frames.append(np.stack(fr))
    init = ttg._init_boxes()
    tr = None
    prev, counts = [None, None], []
    for t, fr in enumerate(frames):
        need = [True, True] if t == 0 else tr.needs_detection.tolist()
        m.set_banks(banks)
        try:
            if tr is None:
                tr = tracking.PoseTracker(m, K, corners, object_ids=[0, 1])
            got = tr.step(fr, init_bbox=[init[b] if need[b] else None for b in range(2)])
        finally:
            m.clear_bank()
        # the same step from one-object calls: crop at the box of the object's own corners, match
        # the crop against that object alone, one batched PnP over both frames (the tracker's seeds)
        boxes = [init[b] if need[b] else tracking.bbox_from_pose(K[b], prev[b], corners[b]) for b in range(2)]
        crops = tracking.crop_resize_batched(fr, np.stack(boxes), ttg.CROP)
        outs = []
        for b in range(2):
            m.set_bank(*banks[b])
            d = {"query_image": crops[b:b + 1]}
            m(d)
            outs.append(d)
        m.clear_bank()
        Kc = np.stack([tracking.crop_K(boxes[b], K[b], ttg.CROP) for b in range(2)])
        m_bids = torch.cat([torch.full_like(o["m_bids"], b) for b, o in enumerate(outs)])
        r = pnp.ransac_pnp_batched(m_bids, torch.cat([o["mkpts_3d_db"] for o in outs]),
                                   torch.cat([o["mkpts_query_f"] for o in outs]),
                                   torch.as_tensor(Kc, dtype=torch.float32).cuda(), reprojection_error=7,
                                   solver="colmap")
        for b in range(2):
            g = got[b]
            assert not g["needs_detection"]
            assert np.array_equal(g["bbox"], boxes[b]) and torch.equal(g["crop"], crops[b:b + 1]), (t, b)
            for k in ("mkpts_3d_db", "mkpts_query_f"):
                assert torch.equal(g[k], outs[b][k]), (t, b, k)
            assert np.array_equal(g["pose"], r["pose"][b].double().cpu().numpy()), (t, b)
            prev[b] = g["pose"]
        counts.append([len(g["inliers"]) for g in got])
    print("inliers per frame and object:", counts)
    assert min(counts[0]) >= 20     # both objects are found: the later frames are tracked, not re-detected


# ------------------------------------------------------------------------------------------------
# kernel-level checks of the new arguments
# ------------------------------------------------------------------------------------------------
def _operands(B, N, S, n_rows, seed=0):
    """fp32 a [B, N, 256] / b [B, S, 256] and their fp16x3 planes; rows l >= n_rows[b] of a are a
    large constant vector along the direction every column of b shares, so they would dominate every
    column's lse and win every column's max if a kernel read them."""
    g = torch.Generator().manual_seed(seed)
    a = 0.3 * torch.randn(B, N, 256, generator=g)
    b = 0.5 + 0.1 * torch.randn(B, S, 256, generator=g)
    for i, n in enumerate(n_rows):
        a[i, n:] = 4.0
    a16, b16 = ops.to_planes(a, True).cuda(), ops.to_planes(b, True).cuda()
    return ops.from_planes(a16, True).double().cpu(), ops.from_planes(b16, True).double().cpu(), a16, b16


def test_lse_conf_colmax_with_row_counts():
    B, N, S = 3, 1000, 1200
    n_rows = [1000, 37, 613]     # frame 1: 30 wholly padded 32-row groups
    a, b, a16, b16 = _operands(B, N, S, n_rows)
    scale = 1.0 / (256 * 0.1)
    dev, f32 = "cuda", torch.float32
    ts, groups = ops.sim_tiles(S), (N + 31) // 32
    buf = lambda *sh, dt=f32: torch.full(sh, float("nan"), device=dev).to(dt) if dt == f32 else \
        torch.zeros(sh, dtype=dt, device=dev)  # noqa: E731
    pm, ps, lse_pt, lse_px = buf(B * N, ts), buf(B * N, ts), buf(B, N), buf(B, S)
    col_m, col_s = buf(B, groups, S), buf(B, groups, S)
    rc = torch.tensor(n_rows, dtype=torch.int32, device=dev)
    ops.sim_lse_cols(a16, b16, B, N, S, 256, scale, pm, ps, lse_pt, col_m, col_s, lse_px, True, row_count=rc)
    conf = torch.full((B, N, S), 7.0, device=dev)
    pv, pi, bv, bi = buf(B * N, ts), buf(B * N, ts, dt=torch.int32), buf(B, N), buf(B, N, dt=torch.int32)
    colmax = buf(B, S, dt=torch.int32)
    ops.sim_conf_colmax(a16, b16, lse_pt, lse_px, conf, B, N, S, 256, scale, pv, pi, bv, bi, colmax, True,
                        row_count=rc)
    torch.cuda.synchronize()
    lse_px, lse_pt, conf = lse_px.cpu().double(), lse_pt.cpu().double(), conf.cpu().double()
    cm = colmax.cpu().view(torch.float32).double()
    for i, n in enumerate(n_rows):
        sim = scale * a[i, :n] @ b[i].T                       # valid rows only
        ref_px = torch.logsumexp(sim, 0)
        ref_pt = torch.logsumexp(sim, 1)
        assert (lse_px[i] - ref_px).abs().max().item() < 1e-4, i
        assert (lse_pt[i, :n] - ref_pt).abs().max().item() < 1e-4, i
        ref_conf = torch.exp(2 * sim - ref_pt[:, None] - ref_px[None])
        assert ((conf[i, :n] - ref_conf).abs() / ref_conf).max().item() < 1e-3, i
        assert (conf[i, n:] == 0).all(), i
        ref_cm = ref_conf.max(0).values
        assert ((cm[i] - ref_cm).abs() / ref_cm).max().item() < 1e-3, i
        # the row maxima of the valid rows (what the match selection reads)
        at = ref_conf.gather(1, bi[i, :n].cpu().long()[:, None])[:, 0]
        assert ((ref_conf.max(1).values - at) / at).max().item() < 1e-3, i


def test_match_select_and_fine_gather_with_bank_of_batch():
    dev = "cuda"
    Kobj, B, N, hc, wc = 3, 4, 600, 12, 16
    S = hc * wc
    bank = torch.tensor([2, 0, 2, 1], dtype=torch.int32, device=dev)
    n_rows = torch.tensor([450, 600, 450, 97], dtype=torch.int32, device=dev)   # n of the frame's object
    g = torch.Generator().manual_seed(1)
    kpts = torch.randn(Kobj, N, 3, generator=g)
    pt_val = 0.2 + 0.8 * torch.rand(B, N, generator=g)
    pt_idx = torch.randint(0, S, (B, N), generator=g, dtype=torch.int32)
    colmax = torch.zeros(B, S, dtype=torch.float32)
    # every row is the maximum of its column; padded rows are the largest of all (they would win)
    for b_ in range(B):
        n = int(n_rows[b_])
        pt_val[b_, n:] += 2.0
        for l in range(N):
            j = int(pt_idx[b_, l])
            colmax[b_, j] = max(colmax[b_, j].item(), pt_val[b_, l].item())
    want = []
    for b_ in range(B):
        for l in range(int(n_rows[b_])):
            j = int(pt_idx[b_, l])
            if pt_val[b_, l] > 0.1 and j // wc >= 2 and j % wc >= 2 and colmax[b_, j] == pt_val[b_, l]:
                want.append((b_, l, j))
    assert want
    cap = B * N
    out = {k: torch.empty(cap, dtype=torch.int64, device=dev) for k in ("b", "i", "j")}
    mconf = torch.empty(cap, device=dev)
    mk3, mkc = torch.empty(cap, 3, device=dev), torch.empty(cap, 2, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    scratch = torch.empty((B * N + 1023) // 1024 + 2, dtype=torch.int32, device=dev)
    ops.match_select_colmax(pt_val.cuda(), pt_idx.cuda(), colmax.view(torch.int32).cuda(), kpts.cuda(), None,
                            B, N, hc, wc, 0.1, 2, 8.0, scratch, out["b"], out["i"], out["j"], mconf, mk3, mkc,
                            count, bank_of_batch=bank, row_count=n_rows)
    M = int(count.item())
    got = list(zip(out["b"][:M].tolist(), out["i"][:M].tolist(), out["j"][:M].tolist()))
    assert got == want
    bb, ii = out["b"][:M].cpu(), out["i"][:M].cpu()
    assert torch.equal(mk3[:M].cpu(), kpts[bank.cpu().long()[bb], ii])
    # fine gather: the descriptor row of each match comes from its frame's object; the windows are
    # those of the per-frame path
    hf, wf = 4 * hc, 4 * wc
    fine = ops.to_planes(torch.randn(B, hf, wf, 128, generator=g), True).cuda()
    desc = torch.randn(Kobj, 128, N, generator=g).cuda()
    x32 = torch.empty(26 * M, 128, device=dev)
    x16 = torch.empty(26 * M, 256, dtype=torch.float16, device=dev)
    ops.fine_gather(fine, desc, out["b"], out["i"], out["j"], x32, x16, M, hf, wf, wc, 4, N, True,
                    bank_of_batch=bank)
    per_frame = desc[bank.long()].contiguous()        # [B, 128, N]: the one-bank-per-frame layout
    r32, r16 = torch.empty_like(x32), torch.empty_like(x16)
    ops.fine_gather(fine, per_frame, out["b"], out["i"], out["j"], r32, r16, M, hf, wf, wc, 4, N, True)
    torch.cuda.synchronize()
    assert torch.equal(x32, r32) and torch.equal(x16, r16)
    assert torch.equal(x32.view(M, 26, 128)[:, 0].cpu(), desc.cpu()[bank.cpu().long()[bb], :, ii])
