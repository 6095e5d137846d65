"""One pose per instance (`uncertainty_pnp_instances`, DESIGN.md §30) by CUDA events.

480x640 scenes of 1, 3 and 6 posed instances (tests/instance_pose_cases.py, sigma 0.03), K = 9 with the centre as the
last keypoint, hn = 256, max_instances = 8, b = 1 and 16.  For each: the device time of `ransac_voting_center` +
`ransac_voting_labels` (covariance 256 x 16) + `uncertainty_pnp_instances` together, of the PnP call alone, and of
`uncertainty_pnp_batched` over all b x 8 rows (the flattened recipe that solves the absent rows too), and of
`refine_poses_instances` (8 rounds, keypoint-anchored, tests/refine_cases.lumpy_mesh) on the PnP poses.  Then the
cost of absent rows: PnP and refinement with num = 1 at I = 8 against I = 1 on the same first-instance inputs.
Median of --iters after 2 warm-ups.  Prints one JSON line per measurement with the card's name and power limit read in the same run; --out
also writes them to a file."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from refine_keypoints import device_ms, gpu_info  # noqa: E402

from pvnet_b200 import extend_utils as eu  # noqa: E402
from pvnet_b200 import ransac_voting_gpu as rv  # noqa: E402
from pvnet_b200 import refine as rfn  # noqa: E402
from tests.instance_pose_cases import K_LINEMOD, POINTS_3D, pose_scene  # noqa: E402
from tests.refine_cases import lumpy_mesh  # noqa: E402

HN, I, THRESH = 256, 8, 0.99


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = gpu_info()
    lines = []

    def emit(d):
        d.update(gpu=name, power_limit=power)
        print(json.dumps(d), flush=True)
        lines.append(d)

    p3 = torch.from_numpy(POINTS_3D).cuda()
    mv, mf = (torch.from_numpy(a).cuda() for a in lumpy_mesh())
    Kd = torch.from_numpy(K_LINEMOD).cuda()
    for n in (1, 3, 6):
        scenes = [pose_scene(n, 2000 + 10 * n + i, sigma=0.03) for i in range(16)]
        for b in (1, 16):
            mask = torch.from_numpy(np.stack([s["mask"] for s in scenes[:b]])).cuda()
            vertex = torch.from_numpy(np.stack([s["field"] for s in scenes[:b]])).cuda()

            def full():
                lab, num = rv.ransac_voting_center(mask, vertex[..., -1, :], HN, THRESH, max_instances=I)
                kp, cov = rv.ransac_voting_labels(lab, vertex, I, HN, THRESH, cov_round_hyp_num=256, cov_min_hyp_num=4096)
                return eu.uncertainty_pnp_instances(kp, num, p3, Kd, cov=cov)
            t_full = device_ms(full, a.iters)
            lab, num = rv.ransac_voting_center(mask, vertex[..., -1, :], HN, THRESH, max_instances=I)
            kp, cov = rv.ransac_voting_labels(lab, vertex, I, HN, THRESH, cov_round_hyp_num=256, cov_min_hyp_num=4096)
            t_pnp = device_ms(lambda: eu.uncertainty_pnp_instances(kp, num, p3, Kd, cov=cov), a.iters)
            kd_rows = Kd.expand(b * I, 3, 3)
            t_flat = device_ms(lambda: eu.uncertainty_pnp_batched(kp.flatten(0, 1), p3, kd_rows, cov=cov.flatten(0, 1)),
                               a.iters)
            poses = eu.uncertainty_pnp_instances(kp, num, p3, Kd, cov=cov)

            def refine():
                return rfn.refine_poses_instances(lab, num, poses, Kd, mv, mf, 0.05, 5.0, keypoints=kp, points_3d=p3,
                                                  cov=cov)
            t_refine = device_ms(refine, max(3, a.iters // 4))
            emit(dict(bench="instance_poses", h=480, w=640, k=9, hn=HN, cov="256x16", max_instances=I, instances=n, b=b,
                      found_mean=float(num.float().mean()), center_labels_pnp_ms=round(t_full, 4),
                      pnp_instances_ms=round(t_pnp, 4), pnp_all_rows_flattened_ms=round(t_flat, 4),
                      refine_instances_8_rounds_ms=round(t_refine, 4)))
            if n == 1:
                one = torch.ones(b, dtype=torch.int32, device="cuda")
                t_i8 = device_ms(lambda: eu.uncertainty_pnp_instances(kp, one, p3, Kd, cov=cov), a.iters)
                kp1, cov1 = kp[:, :1].contiguous(), cov[:, :1].contiguous()
                t_i1 = device_ms(lambda: eu.uncertainty_pnp_instances(kp1, one, p3, Kd, cov=cov1), a.iters)
                p8 = eu.uncertainty_pnp_instances(kp, one, p3, Kd, cov=cov)
                r8 = device_ms(lambda: rfn.refine_poses_instances(lab, one, p8, Kd, mv, mf, 0.05, 5.0),
                               max(3, a.iters // 4))
                r1 = device_ms(lambda: rfn.refine_poses_instances(lab, one, p8[:, :1].contiguous(), Kd, mv, mf, 0.05,
                                                                  5.0), max(3, a.iters // 4))
                emit(dict(bench="instance_poses_absent_rows", b=b, num=1, pnp_I8_ms=round(t_i8, 4),
                          pnp_I1_ms=round(t_i1, 4), refine_I8_ms=round(r8, 4), refine_I1_ms=round(r1, 4)))
    if a.out:
        with open(a.out, "w") as f:
            f.writelines(json.dumps(d) + "\n" for d in lines)


if __name__ == "__main__":
    main()
