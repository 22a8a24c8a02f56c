"""CPU tests: the oracle restatement against the committed golden fixtures (generated from the
unmodified reference: oracle/make_golden.py, oracle/make_reference_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import make_reference_golden, oracle, workload
from tests import golden_io

WEIGHTS = {}


def weights(seed=0):
    if seed not in WEIGHTS:
        WEIGHTS[seed] = workload.synthetic_state_dict(seed)
    return WEIGHTS[seed]


def test_state_dict_layout():
    sd = weights()
    assert len(sd) == 195
    n_params = sum(v.numel() for k, v in sd.items()
                   if "running_" not in k and "num_batches_tracked" not in k)
    assert n_params == 10_226_480  # SURVEY.md App. C


def test_position_encoding_quirk():
    # position_encoding.py:25-28: (-ln(1e4) / d_model // 2) == -1.0 -> div_term = exp(-k), k even
    pe = oracle.position_encoding_sine(256, 8, 8)
    k = torch.arange(0, 128, 2).float()
    x = torch.arange(1, 9).float()
    assert torch.allclose(pe[0::4, 0, :], torch.sin(x[None] * torch.exp(-k)[:, None]), atol=1e-6)
    assert torch.allclose(pe[3::4, :, 0], torch.cos(x[None] * torch.exp(-k)[:, None]), atol=1e-6)


@pytest.mark.parametrize("case", golden_io.cases())
def test_oracle_matches_golden(case):
    data, z = golden_io.load(case)
    stages = {}
    oracle.forward(weights(), data, stages=stages)
    for k in ("b_ids", "i_ids", "j_ids", "m_bids"):
        assert np.array_equal(data[k].numpy(), z[k]), k
    for k, tol in (("mconf", 2e-4), ("mkpts_3d_db", 0), ("mkpts_query_c", 0), ("mkpts_query_f", 2e-3)):
        assert np.allclose(data[k].numpy(), z[k], rtol=0, atol=tol), k
    # expec_f: coordinates tight; the std column is sqrt(clamp(var)) and amplifies 1e-7 to 3e-4
    assert np.allclose(data["expec_f"].numpy()[:, :2], z["expec_f"][:, :2], atol=2e-4)
    assert np.allclose(data["expec_f"].numpy()[:, 2], z["expec_f"][:, 2], atol=5e-3)
    conf = data["conf_matrix"]
    assert np.allclose(conf.max(2).values.numpy(), z["conf_rowmax"], atol=2e-4)
    assert np.allclose(conf.flatten()[torch.from_numpy(z["conf_sample_idx"])].numpy(), z["conf_sample"], atol=2e-4)
    for name, t in (("feat_c", stages["feat_c"]), ("feat_f", stages["feat_f"]),
                    ("tok3d_out", stages["layers"][-1][0]), ("tok2d_out", stages["layers"][-1][1]),
                    ("fine3d_out", stages["fine3d"]), ("fine2d_out", stages["fine2d"])):
        got = t.flatten()[torch.from_numpy(z[name + "_idx"])].numpy()
        assert np.allclose(got, z[name], rtol=1e-3, atol=2e-4), name
    assert float(z["min_thr_margin"]) > 5e-3 and float(z["min_row_margin"]) > 0.05


def test_random_workload_has_no_matches():
    # BASELINE.json config 1 taken literally (random descriptors): no mutual match above thr, M = 0
    data = workload.random_workload(192, 192, 2000)
    oracle.forward(weights(), data)
    assert data["b_ids"].numel() == 0
    assert data["expec_f"].shape == (0, 3)
    assert data["mkpts_query_f"].shape == (0, 2)


def _reference(name):
    return np.load(os.path.join(golden_io.GOLDEN_DIR, "reference", name + ".npz"))


def _close_sampled(t, z, name, atol):
    got = t.flatten()[torch.from_numpy(z[name + "_idx"])].numpy()
    return np.allclose(got, z[name], rtol=0, atol=atol)


@pytest.mark.parametrize("name", list(make_reference_golden.ORACLE_CASES))
def test_oracle_matches_reference_live(name):
    """The oracle against what the unmodified reference computed on the same seeded workload
    (stored by oracle/make_reference_golden.py)."""
    sd, data, cfg = make_reference_golden.oracle_case_inputs(make_reference_golden.ORACLE_CASES[name])
    z = _reference("oracle_" + name)
    d_or = {k: v.clone() for k, v in data.items()}
    oracle.forward(sd, d_or, cfg=cfg)
    conf = d_or["conf_matrix"]
    assert _close_sampled(conf, z, "conf_matrix", 1e-4)
    assert np.allclose(conf.max(2).values.numpy(), z["conf_rowmax"], atol=1e-4)
    assert np.allclose(conf.max(1).values.numpy(), z["conf_colmax"], atol=1e-4)
    if cfg["loftr_coarse"]["attention"] == "full":
        # same weights, different attention: the planted bank no longer matches, compare the raw matrix
        assert np.array_equal(d_or["b_ids"].numpy(), z["b_ids"]) and np.array_equal(d_or["j_ids"].numpy(), z["j_ids"])
        return
    assert len(z["b_ids"]) > 20
    for k in ("b_ids", "i_ids", "j_ids", "m_bids", "mkpts_3d_db", "mkpts_query_c"):
        assert np.array_equal(d_or[k].numpy(), z[k]), k
    assert np.allclose(d_or["mkpts_query_f"].numpy(), z["mkpts_query_f"], atol=2e-3)
    assert np.allclose(d_or["expec_f"][:, :2].numpy(), z["expec_f"][:, :2], atol=2e-4)


def test_pnp_oracle_recovers_planted_poses():
    """oracle/pnp.py (cv2.solvePnPRansac as called by metric_utils.py:169-204, then LM on the inliers)
    on planted frames with 30 % outliers: the refined pose sits at the planted pose up to the noise."""
    import numpy as np
    from oracle import pnp
    b, p3, p2, K, gt = pnp.synthetic_frames(3, outlier_frac=0.3, noise_px=0.5, seed=3)
    for i in range(3):
        m = b == i
        pose, homo, inl, ok = pnp.ransac_pnp(K[i], p2[m], p3[m], pnp_reprojection_error=5)
        assert ok and homo.shape == (4, 4) and 0.6 * m.sum() < len(inl) < 0.8 * m.sum()
        ref = pnp.refined(K[i], p2[m], p3[m], pose, inl)
        assert np.abs(ref - gt[i]).max() < 5e-3 and np.abs(ref - pose).max() < 2e-3


@pytest.mark.parametrize("name", list(make_reference_golden.LOFTR_CASES), ids=list(make_reference_golden.LOFTR_CASES))
def test_loftr_oracle_matches_reference_live(name):
    """oracle/loftr_oracle.py against what the unmodified LoFTR_for_OnePose_Plus
    (src/KeypointFreeSfM/loftr_for_sfm/loftr.py + submodules/LoFTR/src/loftr) computed on a planted
    pair (stored by oracle/make_reference_golden.py)."""
    from oracle import loftr_oracle
    case = make_reference_golden.LOFTR_CASES[name]
    sd, data, cfg = make_reference_golden.loftr_case_inputs(case)
    w, batch = case[1], case[2]
    z = _reference("loftr_" + name)
    d_or = loftr_oracle.forward(sd, {k: v.clone() for k, v in data.items()}, cfg)
    assert len(z["b_ids"]) > 100 * batch
    off = z["i_ids"] - z["j_ids"]
    assert (off == 2 * (w // 8) + 3).mean() > 0.9      # the planted (16, 24) px shift
    for k in ("b_ids", "i_ids", "j_ids", "mkpts0_c", "mkpts1_c"):
        assert np.array_equal(d_or[k].numpy(), z[k]), k
    assert _close_sampled(d_or["conf_matrix"], z, "conf_matrix", 1e-4)
    assert np.allclose(d_or["mconf"].numpy(), z["mconf"], atol=1e-4)
    assert np.allclose(d_or["expec_f"][:, :2].numpy(), z["expec_f"][:, :2], atol=2e-4)
    assert np.allclose(d_or["mkpts1_f"].numpy(), z["mkpts1_f"], atol=2e-3)
    assert np.array_equal(d_or["mkpts0_f"].numpy(), z["mkpts0_f"])
    assert int(z["W"]) == 9
