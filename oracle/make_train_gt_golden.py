"""Writes tests/golden/reference/train_gt.npz: the seeded cases of oracle/train_gt.py:make_case (the
ground-truth list, the matches) and what the UNMODIFIED reference fine_supervision computes on their
dense form, so that the GPU tests need nothing from the reference tree.

    python -m oracle.make_train_gt_golden
"""
import os
import sys

import numpy as np
import torch

from . import train_gt as tg

CASES = {"plain": dict(seed=0, with_scale=False), "scaled": dict(seed=1, with_scale=True)}


def reference_expec(case, window_size=5):
    B, L, S = (int(n) for n in case["shape"])
    fine = torch.full((B, L, S, 2), -50.0)
    fine[case["b_ids"], case["i_ids"], case["j_ids"]] = torch.from_numpy(case["fine_xy"])
    data = {"b_ids": torch.from_numpy(case["m_b"]), "i_ids": torch.from_numpy(case["m_i"]),
            "j_ids": torch.from_numpy(case["m_j"]), "q_hw_c": tuple(int(n) for n in case["hw_c"]),
            "fine_location_matrix_gt": fine}
    if "scale" in case:
        data["query_image_scale"] = torch.from_numpy(case["scale"])
    return tg.reference_fine_supervision(data, tg.config(window_size)).numpy()


def main():
    out = {}
    for name, kw in CASES.items():
        case = tg.make_case(**kw)
        for k, v in case.items():
            out[f"{name}_{k}"] = v
        out[f"{name}_expec_f_gt"] = reference_expec(case)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                        "train_gt.npz")
    np.savez_compressed(path, **out)
    print(f"train_gt -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
