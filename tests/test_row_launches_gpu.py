"""pytest -m gpu: the device-count forward past B * min(N, S) matches.  With the one-pass dual softmax
the value-based mutual test keeps every row of an exact tie (coarse_matching.py:157-165), so a bank
that holds each 3D point twice gives two matches per matched query cell and the match count can
exceed the B * min(N, S) matches the captured fine stage is sized for.  CUDA-graph mode must then
return what the eager forward returns, every tied row included."""
import copy

import pytest
import torch

from oracle import oracle, workload
from tests import parity

pytestmark = pytest.mark.gpu

COPIES = 6     # every 3D point of the bank this many times
THR = 0.005   # below the default 0.1: COPIES tied rows share the softmax over the 3D points


@pytest.fixture(scope="module")
def duplicated_bank():
    """128x160 images (S = 16 x 20 = 320 cells, 252 of them inside the border), a 300-point bank
    planted on every interior cell, then the whole bank repeated COPIES times: N = 1800 > S.  Repeating
    the WHOLE bank leaves the keypoint normalisation (mean, extents) and the linear-attention messages
    unchanged, so rows i, i + 300, ... of the 3D side are the same computation and tie exactly."""
    sd = workload.synthetic_state_dict(0)
    data, _ = workload.planted_workload(sd, 128, 160, 300, 300, batch=2)
    for k in ("keypoints3d", "descriptors3d_db", "descriptors3d_coarse_db"):
        dim = 1 if k == "keypoints3d" else 2
        data[k] = torch.cat([data[k]] * COPIES, dim).contiguous()
    return sd, data


def test_graph_mode_keeps_matches_beyond_fine_capacity(duplicated_bank):
    sd, data = duplicated_bank
    B, N = data["keypoints3d"].shape[:2]
    S = (128 // 8) * (160 // 8)
    cfg = copy.deepcopy(oracle.DEFAULT_CONFIG)
    cfg["coarse_matching"]["thr"] = THR
    ref = {k: v.clone() for k, v in data.items()}
    oracle.forward(sd, ref, cfg=cfg)
    m = parity.cuda_model()
    keys = ("b_ids", "i_ids", "j_ids", "mconf", "expec_f", "mkpts_query_f", "mkpts_3d_db", "mkpts_query_c",
            "conf_matrix")
    try:
        m.coarse_matching.thr = THR
        eager = parity.run_cuda(data)
        M = eager["b_ids"].numel()
        print(f"duplicated bank: N={N} S={S} B={B}: {M} matches, fine capacity B*min(N,S) = {B * min(N, S)}")
        assert M > B * min(N, S), "the workload must produce more matches than the fine stage capacity"
        # every matched cell is matched by all copies of its 3D point (tied rows)
        i, j, b = eager["i_ids"], eager["j_ids"], eager["b_ids"]
        key = (b * N + i % (N // COPIES)) * S + j
        assert set(torch.bincount(key).unique().tolist()) <= {0, COPIES}, "a tied row was dropped"
        rep = parity.compare(eager, ref)
        print("eager vs oracle", rep)
        assert rep["M"] == M
        m.enable_cuda_graphs(True)
        for rnd in range(2):      # capture + replay, then a replay of the cached graph
            g = parity.run_cuda(data)
            for k in keys:
                assert torch.equal(eager[k], g[k]), f"graph mode: {k} differs from eager (round {rnd})"
    finally:
        m.enable_cuda_graphs(False)
        m.coarse_matching.thr = oracle.DEFAULT_CONFIG["coarse_matching"]["thr"]
