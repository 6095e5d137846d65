"""Multi-instance voting (`ransac_voting_center`, DESIGN.md §29) by CUDA events.

480x640 scenes of 1, 3 and 6 planted instances (tests/instance_vote_cases.py, sigma 0.03), K = 9 with the centre
as the last keypoint, hn = 256, max_instances = 8, b = 1 and 16.  For each: the device time of one
`ransac_voting_center` call, of one `ransac_voting_labels` call on its label map (covariance 256 x 16) and of the
two together (median of --iters after 2 warm-ups); and the same work with the API that came before them: the
centre search as a host loop of `pvnet_b200.ransac_voting`'s generate_hypothesis / voting_for_hypothesis per image
and round, as the reference's unfinished function runs them, alone and followed by one `ransac_voting_pipeline`
call per (image, instance) mask.  Prints one JSON line per measurement with the card's name and power limit read in the
same run; --out also writes them to a file."""
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

from pvnet_b200 import ransac_voting as ext  # noqa: E402
from pvnet_b200 import ransac_voting_gpu as rv  # noqa: E402
from tests.instance_vote_cases import instance_scene  # noqa: E402

HN, I, THRESH, MIN_NUM = 256, 8, 0.99, 100


def host_loop(mask, field, idxs):
    """The centre search with the per-image, per-round host loop the reference's function uses."""
    b = mask.shape[0]
    for bi in range(b):
        ys, xs = torch.nonzero(mask[bi], as_tuple=True)
        coords = torch.stack([xs, ys], 1).float()
        direct = field[bi, ys, xs].reshape(-1, 1, 2).contiguous()
        for i in range(I):
            tn = coords.shape[0]
            if tn < MIN_NUM:
                break
            cur = (idxs[bi, i].long() % tn).to(torch.int32).reshape(HN, 1, 2).contiguous()
            hyp = ext.generate_hypothesis(direct, coords, cur)
            inl = torch.zeros([HN, 1, tn], dtype=torch.uint8, device=mask.device)
            ext.voting_for_hypothesis(direct, coords, hyp, inl, THRESH)
            cnt, win = torch.max(torch.sum(inl, 2), 0)
            if int(cnt.item()) < MIN_NUM:
                break
            keep = inl[win[0], 0] == 0
            coords, direct = coords[keep].contiguous(), direct[keep].contiguous()


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

    for n in (1, 3, 6):
        scenes = [instance_scene(n, 1000 + 10 * n + i, sigma=0.03, radius=(35.0, 60.0)) for i in range(16)]
        for b in (1, 16):
            mask = torch.from_numpy(np.stack([s["mask"] for s in scenes[:b]])).cuda()
            vertex = torch.from_numpy(np.stack([s["field"] for s in scenes[:b]])).cuda()
            centre = vertex[..., -1, :]
            idxs = torch.randint(0, 2 ** 31 - 1, (b, I, HN, 2), dtype=torch.int32, device="cuda")
            t_center = device_ms(lambda: rv.ransac_voting_center(mask, centre, HN, THRESH, min_num=MIN_NUM,
                                                                 max_instances=I, idxs=idxs), a.iters)
            labels, num = rv.ransac_voting_center(mask, centre, HN, THRESH, min_num=MIN_NUM, max_instances=I)
            t_labels = device_ms(lambda: rv.ransac_voting_labels(labels, vertex, I, HN, THRESH, cov_round_hyp_num=256,
                                                                 cov_min_hyp_num=4096), a.iters)

            def both():
                lab, _ = rv.ransac_voting_center(mask, centre, HN, THRESH, min_num=MIN_NUM, max_instances=I)
                rv.ransac_voting_labels(lab, vertex, I, HN, THRESH, cov_round_hyp_num=256, cov_min_hyp_num=4096)
            t_both = device_ms(both, a.iters)
            nums = num.cpu().tolist()

            def today():
                host_loop(mask, centre, idxs)
                for bi in range(b):
                    for j in range(nums[bi]):
                        rv.ransac_voting_pipeline(labels[bi:bi + 1] == j + 1, vertex[bi:bi + 1], HN, THRESH,
                                                  cov_round_hyp_num=256, cov_min_hyp_num=4096)
            t_host = device_ms(lambda: host_loop(mask, centre, idxs), max(3, a.iters // 3), warmup=1)
            t_today = device_ms(today, max(3, a.iters // 3), warmup=1)
            emit(dict(bench="instance_voting", h=480, w=640, k=9, hn=HN, cov="256x16", max_instances=I, instances=n,
                      b=b, found_mean=float(np.mean(nums)), center_ms=round(t_center, 4), labels_ms=round(t_labels, 4),
                      center_plus_labels_ms=round(t_both, 4), host_loop_center_ms=round(t_host, 4),
                      host_loop_plus_pipelines_ms=round(t_today, 4)))
    if a.out:
        with open(a.out, "w") as f:
            f.writelines(json.dumps(d) + "\n" for d in lines)


if __name__ == "__main__":
    main()
