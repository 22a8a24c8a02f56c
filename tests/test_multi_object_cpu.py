"""CPU tests of bank sets (several objects in one forward): the C ABI of the new kernel arguments,
the validation of set_banks / object_ids before any launch, the host-side packing of the set
(padding, row counts, row masks) and of one forward's per-frame state, the kernel arguments the
forward passes, and pickling."""
import ctypes
import pickle

import pytest
import torch

from oracle import oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model, _lib, ops
from tests.test_lib_cpu import _stub_ops, header_symbols

NEW = {"opp_sim_lse_cols_rows": "opp_sim_lse_cols", "opp_sim_conf_colmax_rows": "opp_sim_conf_colmax",
       "opp_match_select_colmax_set": "opp_match_select_colmax", "opp_fine_gather_set": "opp_fine_gather"}


def test_new_entry_points_extend_the_old_signatures():
    """Each bank-set entry point is its one-object call with the new pointer arguments inserted
    before the stream (NULL there = the one-object call)."""
    lib = ctypes.CDLL(_lib.LIB_PATH)
    syms = header_symbols()
    P = ctypes.c_void_p
    extra = {"opp_sim_lse_cols_rows": [P], "opp_sim_conf_colmax_rows": [P],
             "opp_match_select_colmax_set": [P, P], "opp_fine_gather_set": [P]}
    for new, old in NEW.items():
        assert new in syms and hasattr(lib, new)
        assert _lib.SIGNATURES[new] == _lib.SIGNATURES[old][:-1] + extra[new] + [P], new
    assert _lib.KERNELS_PER_CALL["opp_match_select_colmax_set"] == 3


class _FakeCuda(torch.Tensor):   # CPU storage that claims to be on a CUDA device (checks only)
    @property
    def is_cuda(self):
        return True


def _fake(t):
    return t.as_subclass(_FakeCuda)


def _model_with_set(ns=(7, 40, 3)):
    m = OnePosePlus_model(oracle.DEFAULT_CONFIG).eval()
    m._bank_set = {"raw": [(torch.rand(1, n, 3), torch.rand(1, 256, n), torch.rand(1, 128, n)) for n in ns],
                   "state": None}
    return m


def test_object_ids_validation_raises_before_any_launch():
    m = _model_with_set()
    img = _fake(torch.rand(3, 1, 64, 64))
    good = {"query_image": img, "object_ids": torch.tensor([2, 0, 1])}
    m._check_inputs(good)
    assert m._check_object_ids(good, 3).tolist() == [2, 0, 1]
    assert m._check_object_ids(dict(good, object_ids=[1, 1, 0]), 3).dtype == torch.int32
    bad = {"missing": None, "length": torch.tensor([0, 1]), "dtype": torch.tensor([0.0, 1.0, 2.0]),
           "bool": torch.tensor([True, False, True]), "range": torch.tensor([0, 3, 1]),
           "negative": torch.tensor([0, -1, 1]), "shape": torch.tensor([[0, 1, 2]])}
    for name, oid in bad.items():
        d = {"query_image": img}
        if oid is not None:
            d["object_ids"] = oid
        with pytest.raises(ValueError):
            m._check_object_ids(d, 3)
    for key, t in (("keypoints3d", torch.rand(3, 7, 3)), ("descriptors3d_db", torch.rand(3, 128, 7)),
                   ("descriptors3d_coarse_db", torch.rand(3, 256, 7))):
        with pytest.raises(ValueError, match="bank set"):
            m._check_inputs(dict(good, **{key: _fake(t)}))
    # object_ids without a set; the forward checks all of this before its first kernel
    m1 = OnePosePlus_model(oracle.DEFAULT_CONFIG).eval()
    with pytest.raises(ValueError, match="no bank set"):
        m1._check_object_ids(good, 3)
    assert m1._check_object_ids({"query_image": img}, 3) is None
    with pytest.raises(ValueError):
        m({"query_image": img, "object_ids": torch.tensor([0, 5, 1])})
    with pytest.raises(NotImplementedError, match="query_image_mask"):
        m({"query_image": img, "object_ids": torch.tensor([0, 1, 1]),
           "query_image_mask": torch.ones(3, 8, 8, dtype=torch.bool)})


def test_train_and_clear_bank():
    m = _model_with_set()
    with pytest.raises(NotImplementedError):
        m.train()
    m.eval()        # train(False) stays allowed
    m.clear_bank()
    assert m._bank is None and m._bank_set is None
    m.train()
    with pytest.raises(NotImplementedError):
        m.set_banks([(torch.rand(1, 5, 3), torch.rand(1, 128, 5))])
    m.eval()
    with pytest.raises(RuntimeError, match="CUDA"):     # the model is on the CPU
        m.set_banks([(torch.rand(1, 5, 3), torch.rand(1, 128, 5))])
    with pytest.raises(ValueError):
        m.set_banks([])


def test_pickling_drops_the_set_state():
    m = _model_with_set()
    m._bank_set["state"] = {"sig": None}
    m2 = pickle.loads(pickle.dumps(m))
    assert m2._bank_set is None and m2._bank is None
    assert m._bank_set is not None


def test_set_packing_and_frame_state(monkeypatch):
    """_encode_bank_set pads every object to N_max (one-object encodings, n_rows, zeros past them);
    _set_frame_state gathers the per-frame state by object id and builds the row counts and the
    uint8 row mask [B*N_max]."""
    calls = []
    _stub_ops(monkeypatch, calls, 4)
    m = _model_with_set(ns=(7, 40, 3))
    m.load_state_dict(workload.synthetic_state_dict(0))
    dev = torch.device("cpu")
    m._plan = m._prepare(dev)
    st = m._resident_set_state()
    assert (st["K"], st["N"]) == (3, 40) and st["n_rows"].tolist() == [7, 40, 3]
    assert st["n_rows"].dtype == torch.int32
    assert st["kpts"].shape == (3, 40, 3) and st["fine"].shape == (3, 128, 40)
    assert st["d3_l0"].shape == (3, 40, 512) and st["l1_mt"].shape == (3, 256, 512) and st["l1_ksum"].shape == (3, 256)
    for k, (kp, _, fine) in enumerate(m._bank_set["raw"]):
        n = kp.shape[1]
        assert torch.equal(st["kpts"][k, :n], kp[0]) and (st["kpts"][k, n:] == 0).all()
        assert torch.equal(st["fine"][k, :, :n], fine[0]) and (st["fine"][k, :, n:] == 0).all()
    # each object encoded alone (its own keypoint statistics): one kpt_encode per object
    assert calls.count("kpt_encode") == 3
    oid = torch.tensor([2, 0, 0, 1], dtype=torch.int32)
    st["l1_ksum"].copy_(torch.arange(3.0)[:, None].expand(3, 256))
    fs = m._set_frame_state(oid, 4)
    assert fs["row_count"].tolist() == [3, 7, 7, 40] and fs["row_count"].dtype == torch.int32
    mask = fs["row_mask"].view(4, 40)
    assert fs["row_mask"].dtype == torch.uint8 and fs["row_mask"].shape == (160,)
    for b, n in enumerate([3, 7, 7, 40]):
        assert mask[b, :n].all() and not mask[b, n:].any()
    assert fs["l1_ksum"][:, 0].tolist() == [2.0, 0.0, 0.0, 1.0]
    assert fs["d3_l0"].shape == (4, 40, 512) and fs["l1_mt"].shape == (4, 256, 512)
    assert fs["bank_of_batch"] is oid and fs["kpts"] is st["kpts"]
    # the forward's stages with the set: masks in the coarse transformer, row counts and object ids
    # in the matching kernels and the fine gather
    recorded = {}

    def rec(name, orig):
        def f(*a, **k):
            recorded.setdefault(name, []).append(k)
            return orig(*a, **k)
        return f
    for name in ("linear_q", "linear_act", "sim_lse_cols", "sim_conf_colmax", "match_select_colmax", "fine_gather"):
        monkeypatch.setattr(ops, name, rec(name, getattr(ops, name)))
    B, S = 4, 96
    q2 = torch.zeros(B, S, 512, dtype=torch.half)
    o2, o3 = m._coarse_transformer(q2, fs, B, S, 40)
    assert o3.shape == (B, 40, 512)
    # every 3D-as-query layer passes the row mask; 3D-as-source K'/V GEMMs do too
    assert sum(k.get("row_mask") is fs["row_mask"] for k in recorded["linear_q"]) == 5
    assert sum(k.get("row_mask") is fs["row_mask"] for k in recorded["linear_act"]) == 4
    out = {}
    count, cap = m._coarse_matching(o2, o3, fs, torch.ones(B, 2), B, 40, 8, 12, 8.0, out)
    assert cap == B * 40
    assert recorded["sim_lse_cols"][0]["row_count"] is fs["row_count"]
    assert recorded["sim_conf_colmax"][0]["row_count"] is fs["row_count"]
    ms = recorded["match_select_colmax"][0]
    assert ms["row_count"] is fs["row_count"] and ms["bank_of_batch"] is oid
    m._fine(torch.zeros(B, 32, 48, 256, dtype=torch.half), fs, (out["b_ids"], out["i_ids"], out["j_ids"],
            out["mkpts_query_c"]), 4, torch.ones(B, 2), 8, 12, (64, 96), out)
    assert recorded["fine_gather"][0]["bank_of_batch"] is oid
    # lazy conf_matrix re-runs the colmax pass with the row counts
    m.conf_matrix_mode = "lazy"
    out = {}
    m._coarse_matching(o2, o3, fs, torch.ones(B, 2), B, 40, 8, 12, 8.0, out)
    n_before = len(recorded["sim_conf_colmax"])
    with torch.no_grad():
        m._materialize_conf(*out["conf_matrix"]._args)
    assert len(recorded["sim_conf_colmax"]) == n_before + 1
    assert recorded["sim_conf_colmax"][-1]["row_count"] is fs["row_count"]


def test_set_layer1_state_is_built_with_the_padded_v_len(monkeypatch):
    """The cached layer-1 3D source state of every object is divided by v_len = N_max, the length
    the set forward's layer-1 query multiplies back by; layer 0 (computed inside the encoding,
    query and state both at N_k) stays at N_k.  A state built at N_k would scale every frame's
    layer-1 message by N_max / N_k."""
    calls = []
    _stub_ops(monkeypatch, calls, 0)
    kv, q = [], []
    monkeypatch.setattr(ops, "kv_state", lambda *a, **k: kv.append((a[6], a[8])))
    real_q = ops.linear_q

    def linear_q(*a, **k):
        q.append(a[6])
        return real_q(*a, **k)
    monkeypatch.setattr(ops, "linear_q", linear_q)
    m = _model_with_set(ns=(7, 40, 3))
    m.load_state_dict(workload.synthetic_state_dict(0))
    m._plan = m._prepare(torch.device("cpu"))
    m._resident_set_state()
    # per object: layer 0 (self, state and query at N_k), then the cached layer-1 state at N_max
    assert kv == [(7, 7), (7, 40), (40, 40), (40, 40), (3, 3), (3, 40)]
    assert q == [7, 40, 3]
    fs = m._set_frame_state(torch.tensor([2, 0], dtype=torch.int32), 2)
    q.clear()
    m._coarse_transformer(torch.zeros(2, 96, 512, dtype=torch.half), fs, 2, 96, 40)
    # layer 0's 2D side (v_len S), then layer 1's 2D side, which reads the cached state: N_max
    assert q[:2] == [96, 40]


def test_tracker_rechecks_the_resident_set():
    from types import SimpleNamespace

    import numpy as np

    from onepose_plus_plus_b200 import tracking
    model = SimpleNamespace(_bank=None, _bank_set={"raw": [0, 1]})
    box = np.zeros((2, 8, 3))
    tr = tracking.PoseTracker(model, np.eye(3), box, object_ids=[1, 0])
    with pytest.raises(ValueError, match="object_ids"):
        tracking.PoseTracker(model, np.eye(3), box, object_ids=[2, 0])
    model._bank_set = {"raw": [0, 1, 2]}       # set_banks with another K after construction
    with pytest.raises(ValueError, match="PoseTracker was built for a set of 2"):
        tr.step(np.zeros((2, 64, 64), np.uint8))
    model._bank_set = None
    with pytest.raises(ValueError, match="no set"):
        tr.step(np.zeros((2, 64, 64), np.uint8))
