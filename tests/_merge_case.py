"""The golden cases of demo.py's cross-class merge (tests/golden/merge_cases.npz) as the reference's own objects: per clip
the rows the merge reads and the merged_result dicts; shared by the CPU and GPU merge tests."""
import numpy as np

CASES = ["demo", "dense", "dense_topk", "big_group", "edges", "zero_area"]
LABELS = [1, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 17, 20, 22, 24, 26, 27, 28, 29, 30, 34, 36, 37, 38, 41, 43, 45,
          46, 47, 48, 49, 51, 52, 54, 56, 57, 58, 59, 60, 61, 62, 63, 64, 65, 66, 67, 68, 69, 70, 72, 73, 74, 76, 77, 78, 79, 80]


def fixture_results(z, name):
    """The reference's merged_result dicts of case `name`, one per clip, in dict order."""
    keys, key_clip, items = z[name + "_keys"], z[name + "_key_clip"], z[name + "_items"]
    out = [{} for _ in z[name + "_nums"]]
    per_clip = [[str(k) for k, c in zip(keys, key_clip) if c == b] for b in range(len(out))]
    for b, k, label, s in items:
        out[int(b)].setdefault(per_clip[int(b)][int(k)], []).append((int(label), np.float32(s)))
    return out


def fixture_rows(z, name):
    """Per clip, the rows the merge reads in scores_list order: (box, class, score)."""
    rows = z[name + "_rows"]
    return [[(r[3:7].copy(), int(r[1]), float(r[2])) for r in rows if int(r[0]) == b] for b in range(len(z[name + "_nums"]))]


def infos(n):
    return [{"video_name": "vid%d" % (b % 2), "fid": 7 + 3 * b} for b in range(n)]


def same_results(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert list(g) == list(w)                      # keys and dict order
        for k in w:
            assert [(l, np.float32(s).tobytes()) for l, s in g[k]] == [(l, s.tobytes()) for l, s in w[k]], k
