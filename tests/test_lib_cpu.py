"""CPU tests of the host side: the C-ABI library loads and exports every symbol declared in
include/opp_b200.h, the drop-in module has the reference's state-dict layout, and the product
fails loudly (no fallback) without a GPU."""
import ctypes
import os
import pickle
import re

import pytest
import torch

from oracle import oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "opp_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(opp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/opp_b200.h but not exported"
    bound = set(_lib.SIGNATURES) | set(_lib.PLAIN)
    assert bound == set(syms), f"ctypes binding and header disagree: {bound ^ set(syms)}"


def test_version_and_tiles_without_gpu():
    lib = _lib.load()
    assert lib.opp_version() >= 100
    g = lib.opp_sim_tiles(100)   # partial slots per column tile = epilogue warp groups (1 or 2)
    assert g in (1, 2) and lib.opp_sim_tiles(4096) == 16 * g and lib.opp_sim_tiles(5000) == 20 * g
    assert lib.opp_kv_chunks(4096) * 256 >= 4096
    assert lib.opp_kv_chunks_b(4096, 64) == lib.opp_kv_chunks(4096)      # enough CTAs: 256-token chunks
    assert lib.opp_kv_chunks_b(4096, 1) == 2 * lib.opp_kv_chunks(4096)   # batch 1: 128-token chunks


def test_state_dict_is_the_reference_layout():
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG)
    sd = workload.synthetic_state_dict(0)
    assert set(m.state_dict().keys()) == set(sd.keys())
    m.load_state_dict(sd, strict=True)
    assert sum(p.numel() for p in m.parameters()) == 10_226_480
    assert "dense_pos_encoding.pe" not in m.state_dict()  # non-persistent, position_encoding.py:35
    m2 = pickle.loads(pickle.dumps(m))  # Ray ships the module object
    assert torch.equal(m2.state_dict()["backbone.conv1.weight"], sd["backbone.conv1.weight"])


def test_position_encoding_matches_oracle():
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG)
    pe = oracle.position_encoding_sine(256, 24, 40)
    assert torch.allclose(m.dense_pos_encoding.pe[0, :, :24, :40], pe, atol=1e-6)


def test_no_cpu_fallback_and_config_errors():
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG).eval()
    data = workload.random_workload(64, 64, 50)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(data)
    import copy
    bad = copy.deepcopy(oracle.DEFAULT_CONFIG)
    bad["loftr_backbone"]["type"] = "VGG"
    with pytest.raises(ValueError):
        OnePosePlus_model(bad)
    bad = copy.deepcopy(oracle.DEFAULT_CONFIG)
    bad["coarse_matching"]["type"] = "sinkhorn"
    with pytest.raises(NotImplementedError):
        OnePosePlus_model(bad)
    bad = copy.deepcopy(oracle.DEFAULT_CONFIG)
    bad["keypoints_encoding"]["type"] = "other"
    with pytest.raises(NotImplementedError):
        OnePosePlus_model(bad)


def test_bn_folding_and_planes_roundtrip():
    from onepose_plus_plus_b200 import ops
    x = torch.randn(7, 64) * 3
    for split in (0, 1):
        back = ops.from_planes(ops.to_planes(x, split), split)
        tol = 2e-6 if split else 2e-3
        assert torch.allclose(back, x, rtol=tol, atol=tol)
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG)
    m.load_state_dict(workload.synthetic_state_dict(0))
    P = m._prepare(torch.device("cpu"))
    sd = m.state_dict()
    w, b = P["layer2.0.conv1"]
    assert w.shape == (208, 2 * 9 * 128) and b.shape == (208,)
    g = sd["backbone.layer2.0.bn1.weight"] / torch.sqrt(sd["backbone.layer2.0.bn1.running_var"] + 1e-5)
    ref = (sd["backbone.layer2.0.conv1.weight"] * g[:, None, None, None]).permute(0, 2, 3, 1).reshape(196, -1)
    got = ops.from_planes(w, 1)[:196]
    assert torch.allclose(got, ref, atol=1e-6)
    assert got.shape[1] == 9 * 128 and ops.from_planes(w, 1)[196:].abs().max() == 0


def _stub_ops(monkeypatch, calls, count_value):
    """Replace every kernel wrapper of ops with a signature-checking recorder (CPU tensors)."""
    import inspect
    from onepose_plus_plus_b200 import ops
    returns_out = {"conv1_gemm": 3, "conv2d_nhwc": 3, "linear_act": 3, "linear_q": 3}

    def stub(name):
        sig = inspect.signature(getattr(ops, name))

        def f(*a, **k):
            bound = sig.bind(*a, **k)
            calls.append(name)
            if name.startswith("match_select"):
                bound.arguments["count"].fill_(count_value)
            if name in returns_out:
                return a[returns_out[name]]
        return f

    names = [n for n, fn in inspect.getmembers(ops, inspect.isfunction)
             if n not in ("to_planes", "from_planes", "_chk", "kv_chunks", "sim_tiles")]
    for n in names:
        monkeypatch.setattr(ops, n, stub(n))
    monkeypatch.setattr(ops, "sim_tiles", lambda c: 2 * ((c + 255) // 256))
    monkeypatch.setattr(ops, "kv_chunks", lambda s_, b_=None: (s_ + 127) // 128)


def test_coarse_matching_host_flow(monkeypatch):
    """Stage sequencing of OnePosePlus_model._coarse_matching with the kernels stubbed out: the
    one-pass dual softmax (lse with column statistics -> conf with column maxima -> match_select);
    every call binds against the real wrapper's signature; conf_matrix follows conf_matrix_mode.
    The flags bench.py reports are fixed: reading them gives True, assigning them raises."""
    calls = []
    _stub_ops(monkeypatch, calls, 0)
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG).eval()
    assert m.coarse_colmax is True and m.coarse_lse_cols is True and m.kv_single_plane is True
    for name in ("coarse_colmax", "coarse_lse_cols", "kv_single_plane"):
        with pytest.raises(AttributeError):
            setattr(m, name, False)
        assert getattr(m, name) is True
    assert m.conf_matrix_mode == "eager"
    B, N, hc, wc = 2, 300, 12, 16
    q2 = torch.zeros(B, hc * wc, 512, dtype=torch.half)
    d3 = torch.zeros(B, N, 512, dtype=torch.half)
    bank = {"Bb": B, "N": N, "kpts": torch.zeros(B, N, 3)}
    for mode in ("eager", "lazy", "skip"):
        m.conf_matrix_mode = mode
        calls.clear()
        out = {}
        count, cap = m._coarse_matching(q2, d3, bank, torch.ones(B, 2), B, N, hc, wc, 8.0, out)
        assert int(count.item()) == 0 and calls == ["sim_lse_cols", "sim_conf_colmax", "match_select_colmax"]
        assert cap == B * N and out["b_ids"].numel() == cap
        if mode == "eager":
            assert out["conf_matrix"].shape == (B, N, hc * wc)
        elif mode == "lazy":
            assert out["conf_matrix"].shape == (B, N, hc * wc) and not torch.is_tensor(out["conf_matrix"])
        else:
            assert out["conf_matrix"] is None


def test_full_forward_host_flow(monkeypatch):
    """Every stage of the forward with all kernels stubbed (CPU tensors): checks the host-side
    sequencing, buffer shapes and wrapper signatures of backbone -> bank encode -> coarse transformer
    -> coarse matching -> fine stage, for a per-image bank and for one shared object."""
    calls = []
    _stub_ops(monkeypatch, calls, 5)
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG).eval()
    m.load_state_dict(workload.synthetic_state_dict(0))
    dev = torch.device("cpu")
    m._plan = m._prepare(dev)
    assert m.kv_single_plane and m._buf("probe_kv16", (8, 512), torch.float16, dev).shape[1] == 512
    B, H, W, N = 2, 64, 96, 200
    img = torch.rand(B, 1, H, W)
    q2, fine_map, (hc, wc) = m._backbone(img)
    S = hc * wc
    assert (hc, wc) == (H // 8, W // 8) and q2.shape == (B, S, 512)
    assert fine_map.shape == (B, H // 2, W // 2, 256)
    # conv1 = im2col + one GEMM chunk; the two FPN upsample-adds are fused into the lateral convs
    assert calls.count("conv2d_nhwc") == 21 and calls.count("conv1_gemm") == 1 and "upsample2x_add" not in calls
    calls.clear()
    # (i) a different object per image: everything per batch element
    bank = m._encode_bank(torch.zeros(B, N, 3), torch.zeros(B, 256, N), torch.zeros(B, 128, N), persistent=False)
    assert calls == ["kpt_encode"] and bank["d3_in"].shape == (B, N, 512) and "d3_l0" not in bank
    calls.clear()
    o2, o3 = m._coarse_transformer(q2, bank, B, S, N)
    assert o2.shape == q2.shape and o3.shape == (B, N, 512)
    # 6 layers x 2 sequences x (kv GEMM, kv_state, q GEMM, Mt+LN, mlp0, mlp2+LN)
    assert calls.count("linear_act") == 24 and calls.count("linear_ln") == 24
    assert calls.count("linear_q") == 12 and calls.count("kv_state") == 12
    # (ii) ONE object for the batch: layer-0 3D side + layer-1 3D source state come from the bank
    calls.clear()
    shared = m._encode_bank(torch.zeros(1, N, 3), torch.zeros(1, 256, N), torch.zeros(1, 128, N), persistent=False)
    assert shared["d3_l0"].shape == (1, N, 512) and shared["l1_mt"].shape == (1, 256, 512)
    assert calls.count("kv_state") == 2 and calls.count("linear_q") == 1
    calls.clear()
    o2, o3 = m._coarse_transformer(q2, shared, B, S, N)
    assert o3.shape == (B, N, 512)
    assert calls.count("kv_state") == 10 and calls.count("linear_q") == 11 and calls.count("linear_ln") == 22
    # workspace: one allocation per name, grown to the high-water mark (bounded memory)
    before = m.workspace_bytes()
    m._coarse_transformer(q2[:, :S // 2].contiguous(), shared, B, S // 2, N)
    assert m.workspace_bytes() == before
    calls.clear()
    out = {}
    count, cap = m._coarse_matching(o2, o3, shared, torch.ones(B, 2), B, N, hc, wc, 8.0, out)
    M = int(count.item())
    assert M == 5 and cap == B * N
    calls.clear()
    m._fine(fine_map, shared, (out["b_ids"], out["i_ids"], out["j_ids"], out["mkpts_query_c"]), M,
            torch.ones(B, 2), hc, wc, img.shape[2:], out)
    assert out["expec_f"].shape == (5, 3) and out["mkpts_query_f"].shape == (5, 2)
    assert calls == ["fine_gather"] + ["linear_act", "fine_attention", "linear_ln", "linear_act", "linear_ln"] * 2 \
        + ["fine_match"]
    data = {}
    m._publish(data, out, M, dev, True)
    assert data["b_ids"].shape == (5,) and data["mkpts_3d_db"].shape == (5, 3) and data["gt_mask"].shape == (5,)
    # empty-match path (fine_preprocess.py:34-37, fine_matching.py:46-55)
    data = {}
    m._publish(data, out, 0, dev, True)
    assert data["expec_f"].shape == (0, 3) and data["mkpts_query_f"].shape == (0, 2)


def test_input_validation_raises_like_the_reference_would():
    """forward() validates batch / point-count / channel shapes before any raw pointer reaches a kernel."""
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG).eval()

    class FakeCuda(torch.Tensor):   # CPU storage that claims to be on a CUDA device (checks only)
        @property
        def is_cuda(self):
            return True

    def fake(t):
        return t.as_subclass(FakeCuda)

    good = {"query_image": fake(torch.rand(2, 1, 64, 64)), "keypoints3d": fake(torch.rand(2, 50, 3)),
            "descriptors3d_db": fake(torch.rand(2, 128, 50)), "descriptors3d_coarse_db": fake(torch.rand(2, 256, 50)),
            "query_image_scale": fake(torch.ones(2, 2))}
    m._check_inputs(good)
    bad_cases = {
        "query_image": fake(torch.rand(2, 3, 64, 64)),
        "keypoints3d": fake(torch.rand(3, 50, 3)),
        "descriptors3d_db": fake(torch.rand(2, 128, 49)),
        "descriptors3d_coarse_db": fake(torch.rand(2, 128, 50)),
        "query_image_scale": fake(torch.ones(1, 2)),
    }
    for key, val in bad_cases.items():
        d = dict(good)
        d[key] = val
        with pytest.raises(ValueError):
            m._check_inputs(d)
    d = dict(good)
    d["query_image"] = fake(torch.rand(2, 1, 60, 64))
    with pytest.raises(ValueError, match="multiples of 8"):
        m._check_inputs(d)
    d = {k: v for k, v in good.items() if k not in ("keypoints3d",)}
    with pytest.raises(KeyError, match="set_bank"):
        m._check_inputs(d)


def test_out_pack_views_and_window_policy():
    """Host logic of the latency mode and of the sparse fine head: the per-match outputs carved out
    of one byte buffer come back as contiguous M-row tensors of the right dtype from a clone, and
    the windows-vs-dense policy switches at the match count where the tile counts cross."""
    from onepose_plus_plus_b200.model import OnePosePlus_model, _OutPack
    cap, fcap = 50, 40
    p = _OutPack(_OutPack.nbytes(cap, fcap), "cpu")
    spec = (("gt_mask", (cap,), torch.bool), ("b_ids", (cap,), torch.int64), ("i_ids", (cap,), torch.int64),
            ("j_ids", (cap,), torch.int64), ("mconf", (cap,), torch.float32), ("mkpts_3d_db", (cap, 3), torch.float32),
            ("mkpts_query_c", (cap, 2), torch.float32), ("expec_f", (fcap, 3), torch.float32),
            ("mkpts_query_f", (fcap, 2), torch.float32))
    t = {k: p.new(k, sh, dt) for k, sh, dt in spec}
    assert p._off <= p.buf.numel()
    g = torch.Generator().manual_seed(0)
    for k, sh, dt in spec:
        if dt == torch.bool:
            t[k].zero_()
        elif dt == torch.int64:
            t[k].copy_(torch.randint(0, 1 << 40, sh, generator=g))
        else:
            t[k].copy_(torch.randn(sh, generator=g))
    for M in (0, 1, 17, 40):
        v = p.views(p.buf.clone(), M)
        for k, sh, dt in spec:
            assert v[k].dtype == dt and v[k].shape == (M,) + tuple(sh[1:]) and v[k].is_contiguous()
            assert torch.equal(v[k], t[k][:M])
    pay = OnePosePlus_model._windows_pay
    # 256x256 fine map: 512 dense M tiles per image and conv; windows: 2 (3) matches per tile
    assert pay(None, 372 * 64, 64, 256, 256) and pay(None, 900, 1, 256, 256)
    assert not pay(None, 1300, 1, 256, 256) and not pay(None, 4096, 1, 256, 256)
