"""GPU: demo.py's cross-class merge on the device (step_b200.postprocess.Merger, step_detect_merge_f32).  Detector + Merger
on the golden histories give the reference's own merged dicts and results.txt bytes (tests/golden/merge_cases.npz); random
cases up to the full 34 x 60 rows per clip equal the numpy restatement (oracle/merge.py) on Detector's own rows; the
result is bit-identical from run to run; StepRunner(detect=dict(..., merge=...)) replays what an eager step computes; a
merge launch does not synchronise."""
import numpy as np
import pytest
import torch

from oracle import merge as om
from step_b200 import synth
from step_b200.postprocess import Detector, Merger, merged_results, result_lines
from _merge_case import CASES, LABELS, fixture_results, fixture_rows, infos, same_results

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def run_case(z, name):
    conf, nms, topk, width, height, thr, valid = z[name + "_cfg"].tolist()
    nums = z[name + "_nums"].tolist()
    prob = torch.from_numpy(z[name + "_prob"]).to(DEV)
    loc = torch.from_numpy(z[name + "_loc"])[:, None].contiguous().to(DEV)          # [R, T=1, 4]: the centre frame
    det = Detector(nums, prob.shape[1], DEV, conf, nms, width, height, topk=max(int(topk), 0))
    d = det.run(prob, loc)
    if not valid:   # rows past valid_tubes (zero-area boxes): the reference's scores_list written straight into det
        rows = fixture_rows(z, name)
        for b, clip in enumerate(rows):
            for k, (box, c, s) in enumerate(clip):
                det.det[b, k] = torch.tensor(list(box) + [s, c, 0, 0], dtype=torch.float32)
            det.count[b] = len(clip)
    merged = Merger(det, thr).run(d)
    return det, d, merged


@pytest.mark.parametrize("name", CASES)
def test_golden_case_equals_reference(golden, name):
    z = golden("merge_cases")
    det, d, merged = run_case(z, name)
    got = merged_results(merged, d, LABELS)
    if z[name + "_cfg"][6]:   # Detector's rows are the reference's scores_list
        rows = det.det.cpu().numpy()
        for b, clip in enumerate(fixture_rows(z, name)):
            assert int(det.count[b]) == len(clip)
            for k, (box, c, s) in enumerate(clip):
                assert np.array_equal(rows[b, k, :4], box) and int(rows[b, k, 5]) == c and rows[b, k, 4] == np.float32(s)
    same_results(got, fixture_results(z, name))
    assert "".join(result_lines(got, infos(len(got)))) == str(z[name + "_text"])


def clustered(rs, B, n, C, people, jitter, conf_lo):
    loc, prob = [], []
    for _ in range(B):
        xy = rs.uniform(0, 260, (people, 2))
        wh = rs.uniform(60, 140, (people, 2))
        who = rs.randint(0, people, n)
        loc.append(np.concatenate([xy[who], xy[who] + wh[who]], 1) + rs.normal(0, jitter, (n, 4)))
        prob.append(rs.uniform(conf_lo, 1, (n, C)))
    return np.concatenate(prob).astype(np.float32), np.concatenate(loc).astype(np.float32)


@pytest.mark.parametrize("seed,B,n,C,people,jitter,conf,nms,topk", [
    (0, 4, 34, 60, 4, 2.0, 0.0, 1.0, 0),       # the full cap: 34 x 60 = 2040 rows per clip
    (1, 8, 34, 60, 3, 1.0, 0.4, 0.4, 0),       # demo.py's thresholds
    (2, 3, 20, 12, 12, 6.0, 0.0, 1.0, 0),      # many groups
    (3, 2, 34, 60, 5, 3.0, 0.01, 0.6, 300),    # top-k 300
    (4, 5, 7, 9, 2, 0.5, 0.2, 0.7, 0),
])
def test_random_cases_equal_oracle(seed, B, n, C, people, jitter, conf, nms, topk):
    rs = np.random.RandomState(seed)
    prob, loc = clustered(rs, B, n, C, people, jitter, 0.0)
    det = Detector([n] * B, C, DEV, conf, nms, 400, 400, topk=topk)
    d = det.run(torch.from_numpy(prob).to(DEV), torch.from_numpy(loc)[:, None].contiguous().to(DEV))
    got = merged_results(Merger(det, 0.8).run(d), d, LABELS)
    rows, count = det.det.cpu().numpy(), det.count.cpu().numpy()
    if seed == 0:
        assert (count == n * C).all()
    for b in range(B):
        clip = [(rows[b, k, :4], int(rows[b, k, 5]), float(rows[b, k, 4])) for k in range(int(count[b]))]
        same_results([got[b]], [om.demo_merge(clip, LABELS, 0.8)])


def test_bit_identical_run_to_run():
    rs = np.random.RandomState(9)
    prob, loc = clustered(rs, 8, 34, 60, 6, 3.0, 0.0)
    det = Detector([34] * 8, 60, DEV, 0.01, 0.6, 400, 400)
    d = det.run(torch.from_numpy(prob).to(DEV), torch.from_numpy(loc)[:, None].contiguous().to(DEV))
    m = Merger(det, 0.8)
    first = {k: v.clone() for k, v in m.run(d).items() if torch.is_tensor(v)}
    for _ in range(5):
        again = m.run(d)
        for k, v in first.items():
            assert torch.equal(again[k], v), k


def valid(m):
    """The defined part of Merger.run's result, per clip: (count, mbox[:keys], pairs[:pairs])."""
    count = m["count"].cpu()
    return [(count[b].tolist(), m["mbox"][b, :count[b, 0]].cpu(), m["pairs"][b, :count[b, 1]].cpu())
            for b in range(count.shape[0])]


def same_valid(a, b):
    assert len(a) == len(b)
    for (ca, ma, pa), (cb, mb, pb) in zip(a, b):
        assert ca == cb and torch.equal(ma, mb) and torch.equal(pa, pb)


def test_step_runner_merge_replays_eager_and_does_not_synchronise():
    import bench
    import step_b200
    B, T_in, HW = 8, 32, 224
    cfg = synth.make_cfg(fp16=True, T=T_in // 4, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(HW, HW))
    nets = bench.build_nets(cfg, DEV)
    tubes = synth.make_proposals(B, 11, cfg.T, HW, HW)
    x = synth.make_clips(B, T_in, HW, HW).to(DEV)
    det = dict(bench.DETECT, merge=0.8)
    eager = step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, use_graph=False, detect=det)
    graph = step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, detect=det)
    plain = step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, use_graph=False, detect=dict(bench.DETECT))
    assert plain.mergers == {} and plain.merged is None
    i = cfg.max_iter - 1
    with torch.no_grad():
        eager(x)
        want = valid(eager.merged[i])
        graph.x.copy_(x)
        torch.cuda.synchronize()
        for _ in range(2):
            torch.cuda.set_sync_debug_mode("error")
            try:
                graph()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            same_valid(valid(graph.merged[i]), want)
    res = merged_results(graph.merged[i], graph.detections[i], LABELS)
    assert sum(len(r) for r in res) > 0
    rows, count = graph.detections[i]["det"].cpu().numpy(), graph.detections[i]["count"].cpu().numpy()
    for b in range(B):
        clip = [(rows[b, k, :4], int(rows[b, k, 5]), float(rows[b, k, 4])) for k in range(int(count[b]))]
        same_results([res[b]], [om.demo_merge(clip, LABELS, 0.8)])


def test_merge_run_does_not_synchronise():
    rs = np.random.RandomState(4)
    prob, loc = clustered(rs, 4, 34, 60, 4, 2.0, 0.0)
    det = Detector([34] * 4, 60, DEV, 0.4, 0.4, 400, 400)
    p, l = torch.from_numpy(prob).to(DEV), torch.from_numpy(loc)[:, None].contiguous().to(DEV)
    m = Merger(det, 0.8)
    m.run(det.run(p, l))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            m.run(det.run(p, l))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
