"""Generate tests/golden/reference/*.npz: what the UNMODIFIED reference (imported from /root/reference
through oracle/ref_shims.py) computes on the seeded workloads of the reference-comparison tests, so
that those tests compare against it without the reference being present:

    python -m oracle.make_reference_golden

The inputs are not stored: every test regenerates them from their seeds (oracle.workload).  Large
tensors are stored as a seeded sample of their flattened elements (`<name>_idx`, `<name>`) plus row
and column maxima where the test bounds them.
"""
import copy
import os
import sys

import numpy as np
import torch

from . import oracle, ref_shims, workload

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                          "reference")

# tests/test_oracle.py::test_oracle_matches_reference_live
ORACLE_CASES = {
    "small_b2": (96, 128, 300, 120, 2, False, "linear"),
    "baseline_512_n5000": (512, 512, 5000, 3000, 1, False, "linear"),
    "small_b2_query_mask": (96, 128, 300, 120, 2, True, "linear"),
    "small_b2_full_attention": (96, 128, 300, 120, 2, False, "full"),
}
# tests/test_oracle.py::test_loftr_oracle_matches_reference_live
LOFTR_CASES = {"b2": (192, 256, 2, False), "b1_scaled": (256, 320, 1, True)}
# tests/test_train_path_cpu.py
TRAIN_GRADS = ("backbone.conv1.weight", "backbone.layer2.0.bn1.weight", "backbone.layer1_outconv2.3.weight",
               "kpt_3d_pos_encoding.encoder.0.weight", "loftr_coarse.layers.0.q_proj.weight",
               "loftr_coarse.layers.5.mlp.2.weight", "loftr_coarse.layers.3.norm1.bias",
               "loftr_fine.layers.1.merge.weight")


def sample_idx(numel, k, seed=7):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, numel, (min(k, numel),), generator=g)


def put_sampled(out, name, t, k=8192):
    idx = sample_idx(t.numel(), k)
    out[name + "_idx"] = idx.numpy()
    out[name] = t.detach().flatten()[idx].numpy()


def oracle_case_inputs(shape):
    sd = workload.synthetic_state_dict(0)
    h, w, n, npl, batch, masked, attention = shape
    data, _ = workload.planted_workload(sd, h, w, n, npl, batch=batch, seed=5)
    if masked:   # img_pad flow (OnePosePlusModel.py:158): bottom / right of the coarse grid is padding
        data["query_image_mask"] = workload.pad_mask(batch, h // 8, w // 8)
    cfg = copy.deepcopy(oracle.DEFAULT_CONFIG)
    cfg["loftr_coarse"]["attention"] = attention
    return sd, data, cfg


def loftr_case_inputs(case):
    from . import loftr_oracle
    h, w, batch, with_scale = case
    sd, data = workload.planted_loftr(h, w, batch=batch, with_scale=with_scale)
    return sd, data, dict(loftr_oracle.DEFAULT_CONFIG)


def train_batch(sd, masked):
    data, _ = workload.planted_workload(sd, 96, 128, 300, 120, batch=2, seed=5)
    S = (96 // 8) * (128 // 8)
    g = torch.Generator().manual_seed(3)
    gt = torch.zeros(2, 300, S, dtype=torch.bool)
    gt[torch.randint(0, 2, (90,), generator=g), torch.randint(0, 300, (90,), generator=g),
       torch.randint(0, S, (90,), generator=g)] = True
    data["conf_matrix_gt"] = gt
    if masked:
        data["query_image_mask"] = workload.pad_mask(2, 12, 16)
    return data


def train_config():
    cfg = copy.deepcopy(oracle.DEFAULT_CONFIG)
    cfg["coarse_matching"]["train"]["train_pad_num_gt_min"] = 20      # < 0.3 * B * min(L, S) at this size
    return cfg


# The training-path comparison runs the CPU forward and backward on one thread, here and in the test:
# the fp32 reduction order of the CPU kernels then does not depend on the host's core count (the
# soft-argmax of expec_f turns a different summation order into ~1e-5 differences).
TRAIN_THREADS = 1


def train_loss(d):
    # (the std column is sqrt(clamp(var)): ill-conditioned near 0, left out of the gradient check)
    return (d["conf_matrix"] * d["conf_matrix_gt"]).sum() + d["expec_f"][:, :2].pow(2).sum()


def save(name, out):
    path = os.path.join(GOLDEN_DIR, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name} -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


def main():
    assert ref_shims.available(), "needs /root/reference"
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    for name, shape in ORACLE_CASES.items():
        sd, data, cfg = oracle_case_inputs(shape)
        ref = ref_shims.build_reference_model(sd, cfg)
        d = {k: v.clone() for k, v in data.items()}
        with torch.no_grad():
            ref(d)
        out = {k: d[k].numpy() for k in ("b_ids", "i_ids", "j_ids", "m_bids", "mkpts_3d_db", "mkpts_query_c",
                                         "mkpts_query_f", "expec_f", "mconf")}
        conf = d["conf_matrix"]
        put_sampled(out, "conf_matrix", conf, 16384)
        out["conf_rowmax"] = conf.max(2).values.numpy()
        out["conf_colmax"] = conf.max(1).values.numpy()
        save("oracle_" + name, out)
    for name, case in LOFTR_CASES.items():
        sd, data, cfg = loftr_case_inputs(case)
        ref = ref_shims.build_reference_loftr(sd, cfg)
        d = {k: v.clone() for k, v in data.items()}
        with torch.no_grad():
            ref(d)
        out = {k: d[k].numpy() for k in ("b_ids", "i_ids", "j_ids", "mkpts0_c", "mkpts1_c", "mconf", "expec_f",
                                         "mkpts0_f", "mkpts1_f")}
        out["W"] = np.int64(d["W"])
        put_sampled(out, "conf_matrix", d["conf_matrix"], 16384)
        save("loftr_" + name, out)
    # LoFTR_for_OnePose_Plus state-dict layout and its positional-encoding buffer
    from . import loftr_oracle
    ref = ref_shims.build_reference_loftr(workload.synthetic_loftr_state_dict(0), dict(loftr_oracle.DEFAULT_CONFIG))
    rs = ref.state_dict()
    out = {"keys": np.array(sorted(rs)), "shapes": np.array([str(tuple(rs[k].shape)) for k in sorted(rs)])}
    put_sampled(out, "pe", ref.pos_encoding.pe, 4096)
    out["pe_shape"] = np.array(ref.pos_encoding.pe.shape)
    save("loftr_layout", out)
    # training-mode forward + backward (tests/test_train_path_cpu.py)
    threads = torch.get_num_threads()
    torch.set_num_threads(TRAIN_THREADS)
    for masked in (False, True):
        sd = workload.synthetic_state_dict(0)
        ref = ref_shims.build_reference_model(sd, train_config()).train()
        d = {k: v.clone() for k, v in train_batch(sd, masked).items()}
        torch.manual_seed(11)
        ref(d)
        loss = train_loss(d)
        ref.zero_grad()
        loss.backward()
        out = {k: d[k].detach().numpy() for k in ("b_ids", "i_ids", "j_ids", "gt_mask", "m_bids", "mkpts_3d_db",
                                                  "mkpts_query_c", "mconf", "mkpts_query_f", "expec_f")}
        put_sampled(out, "conf_matrix", d["conf_matrix"], 16384)
        out["loss"] = np.float64(loss.item())
        params = dict(ref.named_parameters())
        for i, pname in enumerate(TRAIN_GRADS):
            grad = params[pname].grad
            put_sampled(out, f"grad{i}", grad, 4096)
            out[f"grad{i}_absmax"] = np.float32(grad.abs().max().item())
        out["bn_running_mean"] = dict(ref.named_buffers())["backbone.layer1.0.bn1.running_mean"].numpy()
        save("train_masked" if masked else "train", out)
    torch.set_num_threads(threads)


if __name__ == "__main__":
    sys.exit(main())
