"""Depth-anchored refinement per instance (`refine_poses_depth_instances`, DESIGN.md §31) by CUDA events.

480x640 scenes with LINEMOD K of 1, 3 and 6 overlapping `tests/refine_cases.lumpy_mesh(5)` instances (20 480 faces)
0.50-0.56 m away, composited by depth into a label map (tests/refine_depth_instance_cases.py), the composite's
nearest depth with 1 mm of noise as the sensor, a 3 cm gate, L = 8, b = 1 and 16, starts 3 degrees and 1 cm off.
For each: the device time of 8 and of 0 rounds; the same work as a host loop of `refine_poses_depth` on
`labels == j+1` over the present instances, `num` read on the host; and the mean rotation, translation and
optical-axis errors of the start, of keypoint-anchored `refine_poses_instances` (9 model points, 1 px noise) and of
that followed by `refine_poses_depth_instances`.  Then the cost of absent rows: num = 1 at L = 8 against L = 1.
Median of --iters after 2 warm-ups.  Prints one JSON line per measurement with the card's name and power limit read
in the same run; --out also writes them to a file."""
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

from pvnet_b200 import refine as rfn  # noqa: E402
from tests import refine_cases as rf  # noqa: E402
from tests import refine_depth_cases as rdc  # noqa: E402
from tests import refine_depth_instance_cases as ric  # noqa: E402

H, W, L = 480, 640, 8
XS = (-0.16, -0.09, -0.03, 0.03, 0.09, 0.16)
ZS = (0.50, 0.53, 0.51, 0.55, 0.52, 0.56)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = gpu_info()
    lines = []

    def emit(d):
        d.update(gpu=name, power_limit=power)
        print(json.dumps(d), flush=True)
        lines.append(d)

    mesh = rf.lumpy_mesh(5)
    v, f = (torch.from_numpy(x).cuda() for x in mesh)
    K = ric.linemod_k(H, W)
    Kd = torch.from_numpy(K).cuda()
    pts = mesh[0][::1024][:9]
    render = rf.device_depth()
    for n in (1, 3, 6):
        labs, obs, Pt, P0, kps = [], [], [], [], []
        for i in range(16):
            rng = np.random.default_rng(3000 + 10 * n + i)
            P = ric.poses_at(XS[:n], ZS[:n], rng)
            lab, ob = ric.composite(render, mesh, K, P, H, W, rng=rng)
            start = rf.perturb(P, rng, deg=3.0, dist=0.01)
            kp = np.stack([np.stack(rf.rfo.project(pts.astype(np.float64), p, K), -1) for p in P])
            pad = L - n
            labs.append(lab)
            obs.append(ob)
            Pt.append(P)
            P0.append(np.concatenate([start, np.tile(np.eye(3, 4), (pad, 1, 1))]))
            kps.append(np.concatenate([kp + rng.normal(0, 1.0, kp.shape), np.zeros((pad, 9, 2))]))
        for b in (1, 16):
            lab = torch.from_numpy(np.stack(labs[:b])).cuda()
            dep = torch.from_numpy(np.stack(obs[:b])).cuda()
            p0 = torch.from_numpy(np.stack(P0[:b])).cuda()
            num = torch.full((b,), n, dtype=torch.int32, device="cuda")
            args = (lab, num, dep, p0, Kd, v, f, rf.NEAR, rf.FAR, rdc.GATE)
            t8 = device_ms(lambda: rfn.refine_poses_depth_instances(*args), a.iters)
            t0 = device_ms(lambda: rfn.refine_poses_depth_instances(*args, rounds=0), a.iters)

            def host_loop():
                counts = num.tolist()
                for i in range(b):
                    for j in range(counts[i]):
                        rfn.refine_poses_depth((lab[i] == j + 1)[None], dep[i][None], p0[i, j][None], Kd, v, f,
                                               rf.NEAR, rf.FAR, rdc.GATE)
            th = device_ms(host_loop, a.iters)
            emit(dict(bench="refine_depth_instances", h=H, w=W, faces=int(mesh[1].shape[0]), L=L, instances=n, b=b,
                      rounds8_ms=round(t8, 3), rounds0_ms=round(t0, 3), host_loop_8_rounds_ms=round(th, 3)))
            # accuracy: start, keypoint-anchored on the label map, then depth per instance
            kp = torch.from_numpy(np.stack(kps[:b])).float().cuda()
            wgt = torch.tensor([1.0, 0.0, 1.0], device="cuda").expand(b, L, 9, 3).contiguous()
            anchored = rfn.refine_poses_instances(lab, num, p0, Kd, v, f, rf.NEAR, rf.FAR, keypoints=kp,
                                                  points_3d=torch.from_numpy(pts).cuda(), weights_2d=wgt)
            refined, info = rfn.refine_poses_depth_instances(lab, num, dep, anchored, Kd, v, f, rf.NEAR, rf.FAR,
                                                             rdc.GATE, return_info=True)
            errs = {}
            for stage, Q in (("start", p0), ("keypoints", anchored), ("keypoints_depth", refined)):
                Q = Q.cpu().numpy()
                e = np.array([(*rf.pose_error(Q[i, j], Pt[i][j]), abs(Q[i, j, 2, 3] - Pt[i][j][2, 3]))
                              for i in range(b) for j in range(n)])
                errs[stage] = dict(rot_deg=round(float(e[:, 0].mean()), 3),
                                   trans_mm=round(1e3 * float(e[:, 1].mean()), 3),
                                   axis_mm=round(1e3 * float(e[:, 2].mean()), 3))
            st = info["status"][:, :n].cpu().numpy()
            rose = int((info["dist_after"][:, :n] > info["dist_before"][:, :n]).sum())
            emit(dict(bench="refine_depth_instances_accuracy", instances=n, b=b, errors=errs,
                      statuses=sorted(set(st.reshape(-1).tolist())), rows_whose_mean_rose=rose))
        # absent rows: num = 1 at L = 8 against L = 1, on the first instance of each image
        for b in (1, 16) if n == 1 else ():
            lab = torch.from_numpy(np.stack(labs[:b])).cuda()
            dep = torch.from_numpy(np.stack(obs[:b])).cuda()
            p0 = torch.from_numpy(np.stack(P0[:b])).cuda()
            one = torch.ones(b, dtype=torch.int32, device="cuda")
            r8 = device_ms(lambda: rfn.refine_poses_depth_instances(lab, one, dep, p0, Kd, v, f, rf.NEAR, rf.FAR,
                                                                    rdc.GATE), a.iters)
            p1 = p0[:, :1].contiguous()
            r1 = device_ms(lambda: rfn.refine_poses_depth_instances(lab, one, dep, p1, Kd, v, f, rf.NEAR, rf.FAR,
                                                                    rdc.GATE), a.iters)
            emit(dict(bench="refine_depth_instances_absent_rows", instances=n, b=b, num=1, L8_ms=round(r8, 3),
                      L1_ms=round(r1, 3)))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.writelines(json.dumps(d) + "\n" for d in lines)


if __name__ == "__main__":
    main()
