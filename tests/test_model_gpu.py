"""pytest -m gpu: end-to-end parity of the CUDA OnePosePlus_model (called through its public
forward(data) API -> C ABI) against (i) the golden fixtures produced by the unmodified reference
and (ii) the CPU oracle on seeded planted workloads, plus size-independent properties at the
BASELINE sizes."""
import numpy as np
import pytest
import torch

from oracle import oracle, workload
from tests import golden_io, parity

pytestmark = pytest.mark.gpu


def _sd():
    return workload.synthetic_state_dict(0)


@pytest.mark.parametrize("case", golden_io.cases())
def test_golden_parity(case):
    data, z = golden_io.load(case)
    got = parity.run_cuda(data)
    rep = parity.compare(got, {k: z[k] for k in z.files}, max_borderline=0)
    print(case, rep)
    conf = got["conf_matrix"].cpu()
    assert np.allclose(conf.max(2).values.numpy(), z["conf_rowmax"], atol=1e-3)
    assert np.allclose(conf.max(1).values.numpy(), z["conf_colmax"], atol=1e-3)
    assert np.allclose(conf.flatten()[torch.from_numpy(z["conf_sample_idx"])].numpy(), z["conf_sample"], atol=1e-3)
    assert got["m_bids"].cpu().tolist() == z["m_bids"].tolist()
    assert tuple(got["q_hw_c"]) == tuple(s // 8 for s in data["query_image"].shape[2:])
    assert got["W"] == 5 and got["bs"] == data["query_image"].shape[0]


@pytest.mark.parametrize("shape", [(512, 512, 5000, 3000, 1, True),    # BASELINE configs[0]/[1]
                                   (480, 640, 20000, 6000, 1, True),   # BASELINE configs[4]: 640x480, 20k points
                                   (480, 640, 2500, 1500, 1, False),   # config 5 image shape (S = 4800)
                                   (256, 320, 1500, 700, 3, True),
                                   (192, 264, 1501, 500, 2, False)])    # odd point count, 24x33 cells
def test_planted_parity_vs_oracle(shape):
    h, w, n, npl, B, with_scale = shape
    sd = _sd()
    data, meta = workload.planted_workload(sd, h, w, n, npl, batch=B, with_scale=with_scale)
    ref = {k: v.clone() for k, v in data.items()}
    oracle.forward(sd, ref)
    got = parity.run_cuda(data)
    rep = parity.compare(got, ref)
    print(shape, rep)
    assert rep["M"] >= 50 * B
    assert (got["conf_matrix"].cpu() - ref["conf_matrix"]).abs().max().item() <= 1e-3


def test_bench_batch_parity_vs_oracle():
    """BASELINE configs[2], the shape bench.py times: 64 images 512x512 against a shared 5000-point
    bank.  Images 0, 31 and 63 of the batched CUDA forward are compared with the oracle run on each
    image alone (images are independent), conf_matrix rows included."""
    sd = _sd()
    B = 64
    data, _ = workload.planted_workload(sd, 512, 512, 5000, 3000, batch=B)
    got = parity.run_cuda(data)
    assert got["conf_matrix"].shape == (B, 5000, 4096)
    counts = torch.bincount(got["b_ids"].cpu(), minlength=B)
    assert counts.min().item() >= 30, "every image of the bench batch must produce matches"
    for b in (0, 31, 63):
        ref = {k: v[b:b + 1].clone() for k, v in data.items()}
        oracle.forward(sd, ref)
        rep = parity.compare(parity.select_image(got, b), ref)
        print("bench batch image", b, rep)
        assert (got["conf_matrix"][b].cpu() - ref["conf_matrix"][0]).abs().max().item() <= 1e-3


def test_distinct_objects_per_batch_element():
    """Every batch element is a different object (own image, keypoint cloud with its own extents,
    descriptor banks, image scale): exercises desc[b] / kpts[b] / img_scale[b] indexing and the
    batch-0-extents quirk of normalize_3d_keypoints (normalize.py:16-26)."""
    sd = _sd()
    data = workload.hetero_workload(sd, 256, 320, 1500, 700, batch=3)
    ref = {k: v.clone() for k, v in data.items()}
    oracle.forward(sd, ref)
    got = parity.run_cuda(data)
    rep = parity.compare(got, ref)
    print("hetero", rep)
    assert torch.bincount(got["b_ids"].cpu(), minlength=3).min().item() >= 30
    assert (got["conf_matrix"].cpu() - ref["conf_matrix"]).abs().max().item() <= 1e-3


def test_resident_bank_uint8_and_lazy_conf_are_bit_identical():
    """Extensions of the input path (SURVEY §8 f2): set_bank() residency, [1, N, .] banks, uint8
    images with /255 folded into conv1, conf_matrix modes.  All must reproduce the reference-API
    call bit for bit."""
    sd = _sd()
    B = 3
    data, _ = workload.planted_workload(sd, 256, 320, 1500, 700, batch=B)
    img8 = (data["query_image"] * 255).round().clamp(0, 255).to(torch.uint8)
    data["query_image"] = img8.float() / 255      # what data_io.py:107 hands the reference
    base = parity.run_cuda(data)
    keys = ("b_ids", "i_ids", "j_ids", "mconf", "expec_f", "mkpts_query_f", "mkpts_3d_db", "conf_matrix")
    m = parity.cuda_model()

    def run(d):
        d = {k: v.cuda() for k, v in d.items()}
        m(d)
        torch.cuda.synchronize()
        return d

    one = {k: (v[:1] if k in ("keypoints3d", "descriptors3d_db", "descriptors3d_coarse_db") else v)
           for k, v in data.items()}
    a = run(one)                                   # bank given once as [1, N, .]
    u8 = dict(one)
    u8["query_image"] = img8
    b = run(u8)                                    # uint8 frames
    try:
        m.set_bank(one["keypoints3d"], one["descriptors3d_db"], one["descriptors3d_coarse_db"])
        c = run({"query_image": img8, "query_image_scale": data["query_image_scale"]})
        c2 = run({"query_image": img8, "query_image_scale": data["query_image_scale"]})   # cached state
        m.conf_matrix_mode = "lazy"
        d = run({"query_image": img8, "query_image_scale": data["query_image_scale"]})
        lazy = d["conf_matrix"]
        assert not torch.is_tensor(lazy) and lazy.shape == base["conf_matrix"].shape
        d["conf_matrix"] = lazy.materialize()
        m.conf_matrix_mode = "skip"
        e = run({"query_image": img8, "query_image_scale": data["query_image_scale"]})
        assert "conf_matrix" not in e
        m.conf_matrix_mode = "lazy"
        old = run({"query_image": img8, "query_image_scale": data["query_image_scale"]})["conf_matrix"]
        run({"query_image": img8, "query_image_scale": data["query_image_scale"]})
        with pytest.raises(RuntimeError, match="stale"):
            old.materialize()     # the workspace it points into belongs to a later forward
    finally:
        m.conf_matrix_mode = "eager"
        m.clear_bank()
    for name, other in (("[1,N] bank", a), ("uint8", b), ("set_bank", c), ("set_bank cached", c2), ("lazy conf", d)):
        for k in keys:
            assert torch.equal(base[k], other[k]), f"{name}: {k} differs from the reference-API call"
    for k in keys[:-1]:
        assert torch.equal(base[k], e[k]), f"skip conf: {k}"


def test_query_image_mask_parity_vs_oracle():
    """img_pad data flow (OnePosePlusModel.py:158-167, linear_attention.py:49-53,
    coarse_matching.py:108-114): padded coarse cells are zeroed in Q / K / V of the 2D side and get
    -1e9 in the similarity matrix.  Distinct valid rectangles per batch element."""
    sd = _sd()
    data, _ = workload.planted_workload(sd, 256, 320, 1500, 700, batch=3)
    data["query_image_mask"] = workload.pad_mask(3, 32, 40)
    ref = {k: v.clone() for k, v in data.items()}
    oracle.forward(sd, ref)
    got = parity.run_cuda(data)
    rep = parity.compare(got, ref)
    print("query mask", rep)
    assert rep["M"] >= 100
    conf = got["conf_matrix"].cpu()
    assert (conf - ref["conf_matrix"]).abs().max().item() <= 1e-3
    pad = ~data["query_image_mask"].flatten(1)
    assert conf.transpose(1, 2)[pad].abs().max().item() == 0.0, "padded cells must have conf exactly 0"
    # no match lands on a padded cell, and the mask really changes the result
    assert not pad[got["b_ids"].cpu(), got["j_ids"].cpu()].any()
    plain = parity.run_cuda({k: v for k, v in data.items() if k != "query_image_mask"})
    assert plain["b_ids"].numel() != got["b_ids"].numel() or not torch.equal(plain["mconf"], got["mconf"])


def test_full_attention_config_parity_vs_oracle():
    """`loftr_coarse.attention: "full"` (FullAttention, linear_attention.py:64-95; no shipped config
    selects it): conf_matrix and the match lists against the oracle on the same weights."""
    import copy
    from onepose_plus_plus_b200 import OnePosePlus_model
    sd = _sd()
    cfg = copy.deepcopy(oracle.DEFAULT_CONFIG)
    cfg["loftr_coarse"]["attention"] = "full"
    m = OnePosePlus_model(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    data, _ = workload.planted_workload(sd, 192, 256, 900, 400, batch=2)
    ref = {k: v.clone() for k, v in data.items()}
    oracle.forward(sd, ref, cfg=cfg)
    got = {k: v.cuda() for k, v in data.items()}
    m(got)
    torch.cuda.synchronize()
    assert (got["conf_matrix"].cpu() - ref["conf_matrix"]).abs().max().item() <= 1e-3
    if len(ref["b_ids"]):
        print("full attention", parity.compare(got, ref))
    else:
        assert got["b_ids"].numel() == 0


def test_cuda_graph_mode_is_bit_identical():
    """enable_cuda_graphs(): the captured forward (fine stage at capacity, match count read on the
    device, one sync at the end) returns the same bits as the eager path — per-call banks, resident
    bank, M = 0 — and survives shape changes and replays."""
    sd = _sd()
    m = parity.cuda_model()
    keys = ("b_ids", "i_ids", "j_ids", "mconf", "expec_f", "mkpts_query_f", "mkpts_3d_db", "mkpts_query_c",
            "conf_matrix")
    cases = [workload.planted_workload(sd, 512, 512, 5000, 3000, batch=1)[0],
             workload.planted_workload(sd, 256, 320, 1500, 700, batch=3)[0],
             workload.random_workload(192, 192, 2000)]
    eager = [parity.run_cuda(d) for d in cases]
    try:
        m.enable_cuda_graphs(True)
        for rep in range(2):            # second round replays the cached graphs
            for d, e in zip(cases, eager):
                g = parity.run_cuda(d)
                for k in keys:
                    if k in e:
                        assert torch.equal(e[k], g[k]), f"graph mode: {k} differs (round {rep})"
                assert g["gt_mask"].shape == e["gt_mask"].shape and g["W"] == 5
        # outputs are copies: a later replay must not change tensors handed out earlier
        first = parity.run_cuda(cases[0])
        snap = first["mkpts_query_f"].clone()
        other = dict(cases[0])
        other["query_image"] = torch.rand_like(other["query_image"])
        parity.run_cuda(other)
        assert torch.equal(first["mkpts_query_f"], snap)
        # resident bank + uint8 frames under graphs
        d0 = cases[0]
        m.set_bank(d0["keypoints3d"], d0["descriptors3d_db"], d0["descriptors3d_coarse_db"])
        img8 = (d0["query_image"] * 255).round().to(torch.uint8)
        ref = parity.run_cuda({**d0, "query_image": img8.float() / 255})
        m.enable_cuda_graphs(False)
        m.enable_cuda_graphs(True)
        r = {"query_image": img8.cuda(), "query_image_scale": d0["query_image_scale"].cuda()}
        m(r)
        for k in keys[:-1]:
            assert torch.equal(ref[k], r[k]), k
    finally:
        m.enable_cuda_graphs(False)
        m.clear_bank()


def test_fine_windows_path_equals_dense_map():
    """layer1_outconv2 evaluated on the match windows only (fine_windows "sparse") returns the same
    bits as the dense fine map ("dense"), eager and under CUDA graphs; "auto" picks by match count.
    (border_rm keeps matches two cells away from the border, so the zero-padding branch of the
    window kernels is exercised by kernel_checks.check_conv_win, not here.)"""
    sd = _sd()
    m = parity.cuda_model()
    keys = ("b_ids", "i_ids", "j_ids", "mconf", "expec_f", "mkpts_query_f")
    cases = [workload.planted_workload(sd, 512, 512, 5000, 3000, batch=2)[0],
             workload.planted_workload(sd, 480, 640, 3000, 2500, batch=1)[0],
             workload.planted_workload(sd, 64, 96, 900, 60, batch=3)[0]]
    try:
        for d in cases:
            m.fine_windows = "dense"
            dense = parity.run_cuda(d)
            assert dense["b_ids"].numel() > 0
            m.fine_windows = "sparse"
            sparse = parity.run_cuda(d)
            m.enable_cuda_graphs(True)
            graph = parity.run_cuda(d)
            m.enable_cuda_graphs(False)
            m.fine_windows = "auto"
            auto = parity.run_cuda(d)
            for k in keys:
                assert torch.equal(dense[k], sparse[k]), f"sparse windows: {k} differs from the dense map"
                assert torch.equal(dense[k], graph[k]), f"sparse windows under graphs: {k} differs"
                assert torch.equal(dense[k], auto[k]), f"auto: {k} differs"
    finally:
        m.fine_windows = "auto"
        m.enable_cuda_graphs(False)


def test_workspace_is_bounded_across_shapes():
    """Different point counts / image sizes reuse one allocation per buffer name (high-water mark)."""
    m = parity.cuda_model()
    sd = _sd()
    big, _ = workload.planted_workload(sd, 256, 320, 1500, 700, batch=2)
    parity.run_cuda(big)
    hw = m.workspace_bytes()
    for (h, w, n) in ((128, 160, 400), (192, 264, 901), (256, 320, 1499)):
        d, _ = workload.planted_workload(sd, h, w, n, n // 2, batch=2)
        parity.run_cuda(d)
        assert m.workspace_bytes() == hw, "smaller shapes must not allocate"


def test_no_match_path():
    # BASELINE configs[0] taken literally (random descriptors): M = 0, empty outputs, no error
    data = workload.random_workload(192, 192, 2000)
    got = parity.run_cuda(data)
    assert got["b_ids"].numel() == 0 and got["mconf"].numel() == 0
    assert got["expec_f"].shape == (0, 3) and got["mkpts_query_f"].shape == (0, 2)
    assert got["mkpts_3d_db"].shape == (0, 3) and got["conf_matrix"].shape == (1, 2000, 576)
    ref = {k: v.clone() for k, v in data.items()}
    oracle.forward(_sd(), ref)
    assert (got["conf_matrix"].cpu() - ref["conf_matrix"]).abs().max().item() <= 1e-3


def test_properties_at_baseline_size():
    """512x512, 5000 points, batch 4: determinism, ordering, mutual uniqueness, batch independence."""
    sd = _sd()
    data, _ = workload.planted_workload(sd, 512, 512, 5000, 3000, batch=4)
    a = parity.run_cuda(data)
    b = parity.run_cuda(data)
    for k in ("b_ids", "i_ids", "j_ids", "mconf", "expec_f", "mkpts_query_f", "conf_matrix"):
        assert torch.equal(a[k], b[k]), f"{k} is not run-to-run deterministic"
    bi = list(zip(a["b_ids"].tolist(), a["i_ids"].tolist()))
    assert bi == sorted(bi) and len(set(bi)) == len(bi)
    bj = list(zip(a["b_ids"].tolist(), a["j_ids"].tolist()))
    assert len(set(bj)) == len(bj), "a query cell may be matched at most once (mutual NN)"
    assert (a["mconf"] > 0.1).all()
    jy, jx = a["j_ids"] // 64, a["j_ids"] % 64
    assert (jy >= 2).all() and (jx >= 2).all(), "top/left border cells are masked"
    conf = a["conf_matrix"]
    assert conf.min().item() >= 0 and conf.max().item() <= 1.0 + 1e-5
    # image 0 alone gives the same matches as image 0 inside the batch.  Not the same bits: at batch 1
    # the latency tilings are chosen (N-split GEMMs; LayerNorm statistics merged from two column halves
    # across a CTA cluster), so the fp32 rounding of the statistics differs — a tenth of the parity bar
    single = {k: v[:1].clone() for k, v in data.items()}
    s = parity.run_cuda(single)
    m0 = a["b_ids"] == 0
    assert torch.equal(s["i_ids"], a["i_ids"][m0]) and torch.equal(s["j_ids"], a["j_ids"][m0])
    d_conf = (s["mconf"] - a["mconf"][m0]).abs().max().item()
    d_px = (s["mkpts_query_f"] - a["mkpts_query_f"][m0]).abs().max().item()
    print(f"batch independence: |d mconf| {d_conf:.2e}, |d mkpts_query_f| {d_px:.2e} px")
    assert d_conf <= 1e-4 and d_px <= 1e-3


def test_weights_reload_invalidates_plan():
    m = parity.cuda_model(seed=0)
    data, z = golden_io.load("planted_128x160_n400")
    d0 = {k: v.cuda() for k, v in data.items()}
    m(d0)
    sd1 = workload.synthetic_state_dict(1)
    m.load_state_dict(sd1, strict=True)
    d1 = {k: v.cuda() for k, v in data.items()}
    m(d1)
    assert not torch.equal(d0["conf_matrix"], d1["conf_matrix"])
    m.load_state_dict(workload.synthetic_state_dict(0), strict=True)
    d2 = {k: v.cuda() for k, v in data.items()}
    m(d2)
    assert torch.equal(d0["conf_matrix"], d2["conf_matrix"])


def test_fast_fp16_mode_runs_and_is_close():
    data, z = golden_io.load("planted_96x128_n300_b2")
    got = parity.run_cuda(data, precision="fp16")
    conf = got["conf_matrix"].cpu()
    assert np.allclose(conf.max(2).values.numpy(), z["conf_rowmax"], atol=8e-2)
    assert abs(got["b_ids"].numel() - len(z["b_ids"])) <= 5


def test_shared_bank_views_match_materialised_bank():
    """A bank passed as stride-0 expanded views (one object, many images) takes the encode-once
    path; results must equal the per-batch-element path bit for bit."""
    sd = _sd()
    data, _ = workload.planted_workload(sd, 256, 320, 1500, 700, batch=3)
    a = parity.run_cuda(data)
    shared = dict(data)
    for k in ("keypoints3d", "descriptors3d_db", "descriptors3d_coarse_db"):
        shared[k] = data[k][:1].cuda().expand(3, -1, -1)
    shared = {k: (v if v.is_cuda else v.cuda()) for k, v in shared.items()}
    parity.cuda_model()(shared)
    torch.cuda.synchronize()
    for k in ("b_ids", "i_ids", "j_ids", "mconf", "expec_f", "mkpts_query_f", "conf_matrix"):
        assert torch.equal(a[k], shared[k]), k

