"""GPU: the input transform (step_b200.transforms.BaseTransform.apply, kernel step_frames_to_clip_u8) against the reference's
own BaseTransform output (tests/golden/transform_cases.npz): bit-identical to cv2 without IPP, within 1e-4 of the stock
(IPP) wheel relative to the value range; every source form; and the captured StepRunner fed uint8 frames."""
import numpy as np
import pytest
import torch

from oracle import transform as ot
from step_b200 import synth

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def source(z, n):
    """Case n's uint8 BGR frames [T, H0, W0, 3] (cases may share a source)."""
    return z["src_" + str(z[n + "_src"])]


def ipp_on(z, n):
    """Case n's output with cv2's IPP on, stored as int32 bit-pattern offsets from the IPP-off output."""
    return (z[n + "_ipp_off"].view(np.uint32) + z[n + "_ipp_on_ulps"].view(np.uint32)).view(np.float32)


def rgb_frames(src_bgr_hwc):
    return np.ascontiguousarray(src_bgr_hwc[..., ::-1].transpose(0, 3, 1, 2))


def seeded_frames(seed, B, T, H0, W0):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, 256, (B, T, 3, H0, W0)).astype(np.uint8))


def test_golden_cases_bit_identical_to_cv2_without_ipp(golden):
    from step_b200.transforms import BaseTransform
    z = golden("transform_cases")
    worst = {}
    for n in [str(c) for c in z["cases"]]:
        tr = BaseTransform(tuple(z[n + "_size"]), z[n + "_mean"], z[n + "_stds"], int(z[n + "_scale"]))
        frames = torch.from_numpy(rgb_frames(source(z, n)))[None].to(DEV)
        got = tr.apply(frames)[0][:, :, torch.from_numpy(z[n + "_rows"]).to(DEV)].cpu().numpy()
        off, on = z[n + "_ipp_off"], ipp_on(z, n)
        bad = got.view(np.int32) != off.view(np.int32)
        assert not bad.any(), "%s: %d values differ from cv2 (IPP off), first at %s" % (n, bad.sum(), np.argwhere(bad)[0])
        worst[n] = float(np.abs(got - on).max())
        assert worst[n] <= 1e-4 * max(1.0, float(np.abs(on).max())), (n, worst[n])
    print("max |ours - cv2 with IPP| per case: %s" % ", ".join("%s %.3g" % kv for kv in worst.items()))


def test_list_of_mixed_sizes_equals_per_clip_results():
    from step_b200.transforms import BaseTransform
    tr = BaseTransform((400, 400), scale=2)
    sizes = [(360, 640), (360, 480), (361, 641), (200, 300), (800, 800)]
    clips = [seeded_frames(10 + i, 1, 3, h, w)[0].to(DEV) for i, (h, w) in enumerate(sizes)]
    batch = tr.apply(clips)
    assert batch.shape == (len(sizes), 3, 3, 400, 400)
    for i, c in enumerate(clips):
        assert torch.equal(batch[i], tr.apply([c])[0]), sizes[i]
    ref = ot.base_transform(clips[0][:1].cpu().numpy(), (400, 400), scale=2)
    assert np.array_equal(batch[0, :1].cpu().numpy().view(np.int32), ref.view(np.int32))


def test_pinned_host_and_cuda_sources_agree():
    from step_b200.transforms import BaseTransform
    tr = BaseTransform((224, 224), mean=(104, 117, 123), stds=(57.375, 57.12, 58.395), scale=0)
    host = seeded_frames(3, 2, 4, 360, 640).pin_memory()
    a = tr.apply(host)
    b = tr.apply(host.to(DEV))
    c = tr.apply([host[0], host[1]])
    torch.cuda.synchronize()
    assert a.is_cuda and torch.equal(a, b) and torch.equal(a, c)
    ref = ot.base_transform(host[1, 2:].numpy(), (224, 224), (104, 117, 123), (57.375, 57.12, 58.395), 0)
    assert np.array_equal(a[1, 2:].cpu().numpy().view(np.int32), ref.view(np.int32))


def test_strided_sources_equal_the_contiguous_rgb_batch():
    """cv2-layout HWC-BGR frames through a negative channel stride, and the dataset's permuted view (data/ava.py:333-338),
    give the contiguous RGB batch's clip bit for bit."""
    from step_b200 import _lib as L
    from step_b200.transforms import BaseTransform, frame_table
    tr = BaseTransform((400, 400), scale=2)
    T, H0, W0 = 3, 360, 640
    bgr = torch.from_numpy(np.random.RandomState(5).randint(0, 256, (T, H0, W0, 3)).astype(np.uint8)).to(DEV)
    rgb = bgr.flip(-1).permute(0, 3, 1, 2).contiguous()
    want = tr.apply(rgb[None])
    entry = L.step_frame_src(bgr.data_ptr() + 2, H0, W0, H0 * W0 * 3, -1, W0 * 3, 3)
    out = torch.empty_like(want)
    tr.launch(frame_table([entry], torch.device(DEV)), 1, T, out)
    assert torch.equal(out, want)
    assert torch.equal(tr.apply([bgr.flip(-1).contiguous().permute(0, 3, 1, 2)]), want)


def test_fp32_path_basenet_takes_the_transformed_clip():
    import step_b200
    from step_b200.transforms import BaseTransform
    cfg = synth.make_cfg(fp16=False, T=2, max_iter=1, NUM_CHUNKS={1: 1}, image_size=(112, 112))
    net = step_b200.BaseNet(cfg)
    net.load_state_dict(synth.base_net_state_dict(), strict=True)
    net = net.to(DEV).eval()
    x = BaseTransform((112, 112), scale=2).apply(seeded_frames(7, 1, 8, 90, 160).pin_memory())
    with torch.no_grad():
        f = net(x)
    torch.cuda.synchronize()
    assert f.shape[0] == 1 and bool(torch.isfinite(f.float()).all())


def test_step_runner_from_uint8_frames_equals_runner_on_the_clip():
    """C4 shape, graph on: StepRunner(transform=...) fed pinned uint8 frames gives the history and the detections of a
    StepRunner fed the fp32 clip transform.apply returns, bit for bit (the captured kernel, the static uint8 buffer and its
    pinned copy)."""
    import bench
    import step_b200
    from step_b200.transforms import BaseTransform
    B, T_in, HW = 8, 32, 224
    cfg = synth.make_cfg(fp16=True, T=T_in // 4, max_iter=3, NUM_CHUNKS={1: 1, 2: 1, 3: 1}, image_size=(HW, HW))
    nets = bench.build_nets(cfg, torch.device(DEV))
    tubes = synth.make_proposals(B, 11, cfg.T, HW, HW)
    tr = BaseTransform((HW, HW), scale=2)
    frames = seeded_frames(11, B, T_in, 360, 640).pin_memory()
    with pytest.raises(ValueError):
        step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, transform=tr)
    det = dict(bench.DETECT)
    ours = step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, detect=det, transform=tr, source_hw=(360, 640))
    plain = step_b200.StepRunner(cfg, nets, B, T_in, HW, HW, tubes, detect=det)
    with pytest.raises(ValueError):
        ours(seeded_frames(1, B, T_in, 360, 480))

    def snap(d):
        return {k: v.clone() if torch.is_tensor(v) else v for k, v in d.items()}

    with torch.no_grad():
        ho = [snap(h) for h in ours(frames)]
        do = {i: snap(d) for i, d in ours.detections.items()}
        hp = plain(tr.apply(frames))
    torch.cuda.synchronize()
    assert len(ho) == len(hp) == cfg.max_iter
    for a, b in zip(ho, hp):
        assert a.keys() == b.keys()
        for k in a:
            assert torch.equal(a[k], b[k]) if torch.is_tensor(a[k]) else a[k] == b[k], k
    assert do.keys() == plain.detections.keys()
    for i, d in plain.detections.items():
        assert torch.equal(do[i]["count"], d["count"]), i
        for b, n in enumerate(d["count"].tolist()):
            assert torch.equal(do[i]["det"][b, :n], d["det"][b, :n]), (i, b)
    assert int(plain.detections[cfg.max_iter - 1]["count"].sum()) > 0
