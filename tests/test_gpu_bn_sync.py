"""GPU: BatchNorm batch statistics over several ranks (synchronised BatchNorm in the heads of train_step, world_size > 1).

  * per launch, in one process: at every BatchNorm shape of the shipped step, fp16 and fp32, step_bn_stats_local +
    step_bn_stats_merge with one rank give step_bn_stats' outputs bit for bit, and step_bn_bwd_sums + step_bn_bwd_merge_dz
    step_bn_bwd's; with 2..8 ranks holding uneven row ranges of one z / dy (a rank with 1 row, C = 12 on fp32) the merged
    statistics, the running update (against F.batch_norm on the whole) and the gradients are those of the whole in float64
    within the fp32 accumulation bounds of test_gpu_bn_stats.py, and bit-identical from run to run;
  * end to end: tests/_bn_sync_worker.py on two ranks (gloo on cuda:0; with two GPUs also NCCL on cuda:0 and cuda:1) runs
    the shipped fp32 step twice against the DataParallel oracle (_bn_sync_case.py, pinned to the reference by
    test_bn_sync_cpu.py: the reference's ContextNet only takes 25 x 25 maps and has no CPU ROI backward, so its fixture
    starts from conv_feat), unequal rows (3 and 5) against the oracle's (1/W) sum_r L_r, trunk_stats_updated=True, an fp16
    step with a LossScaler, the class-only stage, the cross-rank identity of the averaged gradients and of every running
    statistic, and the refusals."""
import os
import signal
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import _bn_sync_case as sc  # noqa: E402
import _bn_sync_worker as bw  # noqa: E402
from _train_case import rel_l2  # noqa: E402
from test_gpu_bn_affine import shipped_bn_shapes  # noqa: E402,F401  (the fixture)
from test_gpu_bn_stats import U32, n_terms  # noqa: E402
from test_gpu_train_fp32 import TRAIN_TRUNK_L2_TOL  # noqa: E402

pytestmark = pytest.mark.gpu


# ---- the launches --------------------------------------------------------------------------------------------------------
def _operands(f16, M, C, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dt = torch.float16 if f16 else torch.float32
    mu = torch.randn(C, device="cuda", generator=gen) * 2.0
    sig = torch.rand(C, device="cuda", generator=gen) * 1.5 + 0.05
    z = (torch.randn((M, C), device="cuda", generator=gen) * sig + mu).to(dt)
    dy = (torch.randn((M, C), device="cuda", generator=gen) * (1024.0 if f16 else 1.0) * 1e-2).to(dt)
    gamma = torch.rand(C, device="cuda", generator=gen) * 1.5 + 0.1
    beta = torch.randn(C, device="cuda", generator=gen) * 0.5
    rm0 = torch.randn(C, device="cuda", generator=gen) * 0.1
    rv0 = torch.rand(C, device="cuda", generator=gen) + 0.5
    return dict(z=z, dy=dy, gamma=gamma, beta=beta, rm0=rm0, rv0=rv0, gscale=1.0 / 1024.0 if f16 else 1.0)


def _apply(lib, L, f16, z, st):
    M, C = z.shape
    y = torch.empty_like(z)
    apply = lib.step_bn_apply_f16 if f16 else lib.step_bn_apply_f32
    L.check(apply(L.ptr(z), C, M, C, L.ptr(st[2]), L.ptr(st[3]), 1, L.ptr(y), C, C, None, 0, C, None, 0, L.stream()))
    return y


def run_fused(f16, o):
    from step_b200 import _lib as L
    lib = L.lib()
    z, dy = o["z"], o["dy"]
    M, C = z.shape
    rm, rv = o["rm0"].clone(), o["rv0"].clone()
    st = torch.empty((4, C), device="cuda")
    nbytes = lib.step_bn_stats_workspace_bytes(M, C)
    ws = torch.empty((nbytes // 4,), device="cuda")
    stats = lib.step_bn_stats_f16 if f16 else lib.step_bn_stats_f32
    L.check(stats(L.ptr(z), C, M, C, L.ptr(o["gamma"]), L.ptr(o["beta"]), 1e-5, 0.1, L.ptr(rm), L.ptr(rv), L.ptr(st[0]), L.ptr(st[1]),
                  L.ptr(st[2]), L.ptr(st[3]), L.ptr(ws), nbytes, L.stream()))
    y = _apply(lib, L, f16, z, st)
    dz = torch.empty_like(z)
    dg, db = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    nbytes = lib.step_bn_bwd_workspace_bytes(M, C)
    ws = torch.empty((nbytes // 4,), device="cuda")
    bwd = lib.step_bn_bwd_f16 if f16 else lib.step_bn_bwd_f32
    L.check(bwd(L.ptr(dy), C, L.ptr(y), C, L.ptr(z), C, M, C, L.ptr(st[0]), L.ptr(st[1]), L.ptr(o["gamma"]), 1, o["gscale"], L.ptr(dz),
                C, L.ptr(dg), L.ptr(db), L.ptr(ws), nbytes, L.stream()))
    return dict(st=st, rm=rm, rv=rv, y=y, dz=dz, dg=dg[None], db=db[None])


def run_split(f16, o, rows):
    """The ranks' row ranges of z / dy through the local entries, their outputs stacked in rank order, and the merges."""
    from step_b200 import _lib as L
    lib = L.lib()
    z, dy = o["z"], o["dy"]
    M, C = z.shape
    W = len(rows)
    cuts = [0]
    for n in rows:
        cuts.append(cuts[-1] + n)
    assert cuts[-1] == M
    rm, rv = o["rm0"].clone(), o["rv0"].clone()
    trip = torch.full((W, 3, C), float("nan"), device="cuda")
    local = lib.step_bn_stats_local_f16 if f16 else lib.step_bn_stats_local_f32
    for r in range(W):
        nbytes = lib.step_bn_stats_workspace_bytes(rows[r], C)
        ws = torch.full((nbytes // 4,), float("nan"), device="cuda")
        L.check(local(L.ptr(z[cuts[r]:]), C, rows[r], C, L.ptr(trip[r]), C, L.ptr(ws), nbytes, L.stream()))
    st = torch.full((4, C), float("nan"), device="cuda")
    L.check(lib.step_bn_stats_merge(L.ptr(trip), W, C, M, C, L.ptr(o["gamma"]), L.ptr(o["beta"]), 1e-5, 0.1, L.ptr(rm), L.ptr(rv),
                                    L.ptr(st[0]), L.ptr(st[1]), L.ptr(st[2]), L.ptr(st[3]), L.stream()))
    y = _apply(lib, L, f16, z, st)
    sums = torch.full((W, 2, C), float("nan"), device="cuda")
    dg, db = torch.full((W, C), float("nan"), device="cuda"), torch.full((W, C), float("nan"), device="cuda")
    sums_fn = lib.step_bn_bwd_sums_f16 if f16 else lib.step_bn_bwd_sums_f32
    for r in range(W):
        nbytes = lib.step_bn_bwd_sums_workspace_bytes(rows[r], C)
        ws = torch.full((nbytes // 4,), float("nan"), device="cuda")
        L.check(sums_fn(L.ptr(dy[cuts[r]:]), C, L.ptr(y[cuts[r]:]), C, L.ptr(z[cuts[r]:]), C, rows[r], C, L.ptr(st[0]), L.ptr(st[1]), 1,
                        o["gscale"], L.ptr(sums[r]), C, L.ptr(dg[r]), L.ptr(db[r]), L.ptr(ws), nbytes, L.stream()))
    dz = torch.full_like(z, float("nan"))
    merge_dz = lib.step_bn_bwd_merge_dz_f16 if f16 else lib.step_bn_bwd_merge_dz_f32
    nbytes = lib.step_bn_bwd_merge_dz_workspace_bytes(C)
    for r in range(W):
        ws = torch.full((nbytes // 4,), float("nan"), device="cuda")
        L.check(merge_dz(L.ptr(sums), W, C, M, L.ptr(dy[cuts[r]:]), C, L.ptr(y[cuts[r]:]), C, L.ptr(z[cuts[r]:]), C, rows[r], C,
                         L.ptr(st[0]), L.ptr(st[1]), L.ptr(o["gamma"]), 1, L.ptr(dz[cuts[r]:]), C, L.ptr(ws), nbytes, L.stream()))
    return dict(st=st, rm=rm, rv=rv, y=y, dz=dz, dg=dg, db=db)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def assert_bit_equal(a, b, what):
    for k in a:
        assert torch.equal(_bits(a[k]), _bits(b[k])), (what, k)


@pytest.mark.parametrize("f16", [True, False], ids=["f16", "f32"])
def test_one_rank_split_is_the_fused_entries_bit_for_bit(shipped_bn_shapes, f16):  # noqa: F811
    shapes = sorted({(M, C) for M, C, _, _ in shipped_bn_shapes})
    assert len(shapes) >= 10
    for i, (M, C) in enumerate(shapes):
        o = _operands(f16, M, C, seed=i)
        a, b = run_fused(f16, o), run_split(f16, o, [M])
        torch.cuda.synchronize()
        assert_bit_equal(a, b, (M, C))
        torch.cuda.empty_cache()


SPLITS = {
    # name: f16, C, rows per rank
    "w2_one_row": (False, 12, [1, 3000]),
    "w3": (True, 24, [517, 1, 2048]),
    "w4_f32": (False, 36, [4000, 250, 1, 77]),
    "w5": (True, 64, [100, 1, 7, 33000, 12]),
    "w8_many_chunks": (False, 12, [1, 2, 3, 4, 5, 600, 140000, 9]),
    "w8_f16": (True, 8, [300, 1, 1, 2, 9000, 64, 3, 5]),
}


@pytest.mark.parametrize("name", list(SPLITS))
def test_ranks_merge_to_the_whole_in_float64(name):
    f16, C, rows = SPLITS[name]
    M = sum(rows)
    o = _operands(f16, M, C, seed=7)
    r = run_split(f16, o, rows)
    again = run_split(f16, o, rows)
    torch.cuda.synchronize()
    assert_bit_equal(r, again, "run to run")
    V = 8 if f16 else 4
    W = len(rows)
    # each rank's chunked reduction, then W triples merged: at most W + 5 more merges than one rank's bound
    n = max(n_terms(m, C, V) for m in rows) + W + 5
    z = o["z"].double()
    mean, var = z.mean(0), z.var(0, unbiased=False)
    std = var.sqrt()
    mean_d, rstd_d, scale_d, shift_d = r["st"].double()
    assert bool(((mean_d - mean).abs() <= n * U32 * (mean.abs() + std)).all())
    var_d = 1.0 / rstd_d ** 2 - 1e-5
    assert bool(((var_d - var).abs() <= 2 * n * U32 * std * (mean.abs() + std) + 4 * U32 * (var + 1e-5)).all())
    rm_t, rv_t = o["rm0"].clone(), o["rv0"].clone()
    F.batch_norm(o["z"].float(), rm_t, rv_t, o["gamma"], o["beta"], True, 0.1, 1e-5)
    rm_ref = 0.9 * o["rm0"].double() + 0.1 * mean
    rv_ref = 0.9 * o["rv0"].double() + 0.1 * var * M / (M - 1)
    for got, ref, tch in ((r["rm"], rm_ref, rm_t), (r["rv"], rv_ref, rv_t)):
        tol = 0.1 * n * U32 * (mean.abs() + std) * (1 + std) + 4 * U32 * ref.abs()
        assert bool(((got.double() - ref).abs() <= tol).all())
        assert bool(((got.double() - tch.double()).abs() <= 2 * tol + 1e-6 * ref.abs()).all())
    # the backward: each rank's dgamma / dbeta are its own rows' sums; dz uses the sums of all rows
    y = r["y"].double()
    g = o["dy"].double() * (y > 0)
    xhat = (z - mean_d) * rstd_d
    gs = o["gscale"]
    cuts = [0]
    for m in rows:
        cuts.append(cuts[-1] + m)
    sg, sgx = g.sum(0), (g * xhat).sum(0)
    bound_g, bound_gx = 1e-30, 1e-30
    for k in range(W):
        gk, xk = g[cuts[k]:cuts[k + 1]], xhat[cuts[k]:cuts[k + 1]]
        bg = n * U32 * gk.abs().sum(0) + 1e-30
        bgx = n * U32 * (gk * xk).abs().sum(0) * 2 + 1e-30
        assert bool(((r["db"][k].double() - gs * gk.sum(0)).abs() <= gs * bg).all()), k
        assert bool(((r["dg"][k].double() - gs * (gk * xk).sum(0)).abs() <= gs * bgx).all()), k
        bound_g, bound_gx = bound_g + bg, bound_gx + bgx
    a = o["gamma"].double() * rstd_d
    dz_ref = a * (g - sg / M - xhat * sgx / M)
    dzb = a.abs() * (4 * U32 * (g.abs() + (sg / M).abs() + (xhat * sgx / M).abs()) + bound_g / M + xhat.abs() * bound_gx / M
                     + 4 * U32 * xhat.abs() * (sgx / M).abs())
    if f16:
        dzb = dzb + 2.0 ** -11 * dz_ref.abs() + 2.0 ** -24
    assert bool(((r["dz"].double() - dz_ref).abs() <= dzb).all())


# ---- end to end on two ranks ----------------------------------------------------------------------------------------------
def run_worker(backend, out_dir, timeout=1500):
    """The worker under torch.distributed.run in its own session; on a timeout the whole process group is killed, so no
    process outlives the test."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node=2",
           os.path.join(HERE, "_bn_sync_worker.py"), backend, str(out_dir)]
    proc = subprocess.Popen(cmd, cwd=ROOT, env=env, start_new_session=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    try:
        out, _ = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        proc.communicate()
        raise
    assert proc.returncode == 0, out.decode(errors="replace")[-6000:]
    return [torch.load(os.path.join(out_dir, "rank%d.pt" % r)) for r in range(2)]


@pytest.fixture(scope="module")
def gloo(tmp_path_factory):
    return run_worker("gloo", tmp_path_factory.mktemp("gloo"))


def _sds_from(state, base):
    """Oracle state dicts from the device nets' state (parameters) with base's running statistics, trainable as base's."""
    out = {}
    for m, sd in base.items():
        out[m] = {k: (state["%s.%s" % (m, k)].clone().requires_grad_(v.requires_grad) if v.requires_grad
                      else v.detach().clone()) for k, v in sd.items()}
    return out


def check_against_oracle(res, sds, J, losses, what):
    """res: both ranks' results of one step (loss, averaged grads, running statistics after it)."""
    J.backward()
    for rank in (0, 1):
        ref = float(losses[rank].detach())
        assert abs(res[rank]["loss"] - ref) <= 1e-4 * abs(ref), (what, rank)
    n = 0
    for m, sd in sds.items():
        for k, ref in sd.items():
            if ref.grad is None:
                continue
            rel = rel_l2(res[0]["grads"]["%s.%s" % (m, k)], ref.grad)
            # Looser than test_gpu_bn_stats' single-rank bounds (1.5x and 1x): each trunk replica's statistics come from one
            # clip, so a max-pool, ROIPool or ReLU decision near a tie moves a larger share of every channel's gradient.
            # Worst measured on an H100: 2.97e-2 (trunk), 2.38e-2 (heads), with medians of 1.6e-2 and 8e-3;
            # test_shipped_fp32_two_steps_like_the_oracle also checks that the head statistics are the synchronised ones.
            tol = 2.5 * TRAIN_TRUNK_L2_TOL if m in ("base_net", "context_net") else 2.0 * TRAIN_TRUNK_L2_TOL
            assert rel <= tol, (what, m, k, rel)
            n += 1
        for k, v in sd.items():
            if "running_" in k:
                assert rel_l2(res[0]["buffers"]["%s.%s" % (m, k)], v.detach()) <= 1e-4, (what, m, k)
            elif k.endswith("num_batches_tracked"):
                assert int(res[0]["buffers"]["%s.%s" % (m, k)]) == int(v), (what, m, k)
    assert n == len(res[0]["grads"])
    return n


def assert_ranks_identical(res, key):
    a, b = res[0][key], res[1][key]
    for part in ("grads", "buffers"):
        assert a[part].keys() == b[part].keys()
        for k in a[part]:
            assert torch.equal(a[part][k], b[part][k]), (key, part, k)


def test_shipped_fp32_two_steps_like_the_oracle(gloo):
    cfg = sc.case_cfg("ctx", False, False)
    ranks = sc.split_rows(cfg, *sc.whole_case("ctx", cfg))
    sds = sc.oracle_sds("ctx", cfg, 0)
    J, losses, _ = sc.sync_objective(cfg, sds, ranks)
    assert check_against_oracle([r["ship1"] for r in gloo], sds, J, losses, "step 1") > 300
    # the heads' gradients are those of statistics over both ranks' rows, not of each rank's own rows: against an oracle
    # whose heads normalise per rank the same gradients are off by 30% to 100% (measured), against this one by ~1%
    per_rank = []
    for r in range(2):
        s = sc.oracle_sds("ctx", cfg, 0)
        sc.sync_objective(cfg, s, [ranks[r]])[0].backward()
        per_rank.append(s)
    for i in range(3):
        m = "det_net%d" % i
        ks = [k for k, v in sds[m].items() if v.grad is not None]
        synced = sorted(rel_l2(gloo[0]["ship1"]["grads"]["%s.%s" % (m, k)], sds[m][k].grad) for k in ks)
        unsynced = sorted(rel_l2(gloo[0]["ship1"]["grads"]["%s.%s" % (m, k)], (per_rank[0][m][k].grad + per_rank[1][m][k].grad) / 2)
                          for k in ks)
        assert synced[len(ks) // 2] < 0.1 * unsynced[len(ks) // 2], (m, synced[len(ks) // 2], unsynced[len(ks) // 2])
    sds2 = _sds_from(gloo[0]["ship1_state"], sds)
    J, losses, _ = sc.sync_objective(cfg, sds2, ranks)
    check_against_oracle([r["ship2"] for r in gloo], sds2, J, losses, "step 2")
    for key in ("ship1", "ship2"):
        assert_ranks_identical(gloo, key)
        assert not gloo[0][key]["skipped"]
    assert all(int(v) == 2 for k, v in gloo[0]["ship2"]["buffers"].items() if k.endswith("num_batches_tracked"))


def test_unequal_rows_like_the_oracle(gloo):
    cfg = sc.case_cfg("ctx", False, True)
    ranks = [bw.unequal_case(cfg, r) for r in range(2)]
    assert [t.shape[0] for t in ranks[1][1]] == [5, 5, 5]
    sds = sc.oracle_sds("ctx", cfg, 1)
    J, losses, _ = sc.sync_objective(cfg, sds, ranks)
    check_against_oracle([r["unequal"] for r in gloo], sds, J, losses, "unequal rows")
    assert_ranks_identical(gloo, "unequal")


def test_trunk_running_statistics_are_rank_zeros(gloo):
    """After the broadcast both ranks hold what rank 0 computed alone: with trunk_stats_updated=True, rank 0's own
    forward's update; the gradients are those of the step that updated them itself."""
    assert_ranks_identical(gloo, "prepass")
    pre0 = gloo[0]["prepass_buffers"]
    for rank in (0, 1):
        got = gloo[rank]["prepass"]["buffers"]
        for k, v in got.items():
            if k.startswith(("base_net.", "context_net.")):
                assert torch.equal(v, pre0[k]), (rank, k)
    assert any(not torch.equal(gloo[1]["prepass_buffers"][k], pre0[k]) for k in pre0 if k.startswith("base_net.")
               and "running_mean" in k)                               # rank 1's own forward differed
    for k, v in gloo[0]["prepass"]["grads"].items():
        assert torch.equal(v, gloo[0]["ship1"]["grads"][k]), k


def test_fp16_step_with_loss_scaler(gloo):
    assert_ranks_identical(gloo, "fp16")
    r = gloo[0]["fp16"]
    assert not r["skipped"] and r["loss_scale"] == 1024.0
    assert all(bool(torch.isfinite(g).all()) for g in r["grads"].values())
    for k, v in r["buffers"].items():
        if "running_" in k:
            assert not torch.equal(v, gloo[0]["fp16_before"][k]) and bool(torch.isfinite(v).all()), k


def test_class_only_stage_like_the_oracle(gloo):
    cfg = sc.case_cfg("cls", False, False)
    ranks = sc.split_rows(cfg, *sc.whole_case("cls", cfg))
    sds = sc.oracle_sds("cls", cfg, 0)
    J, losses, _ = sc.sync_objective(cfg, sds, ranks, cls_only=True)
    check_against_oracle([r["cls"] for r in gloo], sds, J, losses, "cls")
    assert_ranks_identical(gloo, "cls")


def test_refusals_on_both_ranks(gloo):
    words = {"steps": "number of steps", "loss_scale": "loss scale", "zero_rows": "no rows", "world_size": "world_size=3"}
    for rank in (0, 1):
        ref = gloo[rank]["refusals"]
        for name, w in words.items():
            assert ref[name].startswith("ValueError") and w in ref[name], (rank, name, ref[name])
            assert ref[name + ":unchanged"], (rank, name)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL needs two GPUs (it refuses two ranks on one device)")
def test_nccl_equals_gloo(gloo, tmp_path):
    nccl = run_worker("nccl", tmp_path)
    for key in ("ship1", "ship2", "unequal", "cls", "fp16"):
        assert_ranks_identical(nccl, key)
        for part in ("grads", "buffers"):
            for k, v in nccl[0][key][part].items():
                assert torch.equal(v, gloo[0][key][part][k]), (key, part, k)
