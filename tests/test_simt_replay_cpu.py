"""CPU: the exact replay of tests/_simt_replay.py pinned to exact rational arithmetic.

  * fma32 against a fractions.Fraction evaluation of a * b + c rounded to fp32 by hand (round half to even, subnormals,
    overflow to +-inf, the sign of an exact zero), on random operands and on the cases a float64 shortcut gets wrong:
    exact fp32 midpoints, a sticky bit below a midpoint, total cancellation, subnormal results, signed zeros, overflow;
  * simt_conv_replay of a tiny convolution (2 taps, Cin = 20: a partial 16-channel block, Cout = 3, one padded tap, a
    residual) against a pure-Python loop in the kernel's order, for both storage types;
  * the SASS the replay's epilogue order rests on: when the library's conv_simt.o and cuobjdump are present, the fp32
    instance of conv3d_simt_kernel must still scale, shift, add the residual and clamp in four separately rounded
    instructions (a compiler that contracts them would otherwise show up as a one-ulp mismatch on the GPU)."""
import math
import os
import re
import shutil
import struct
import subprocess
import sys
from fractions import Fraction

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import _simt_replay as S  # noqa: E402

F32_MAX_EXP = 128                # fp32 values are below 2^128
F32_MIN_EXP = -126               # smallest normal exponent; the subnormal quantum is 2^-149


def bits32(v):
    return struct.unpack("<I", struct.pack("<f", v))[0]


def round_f32(q, neg_zero=False):
    """Exact rational q -> the nearest fp32 value (ties to even) as a Python float; +-inf past the largest finite value.
    neg_zero: the sign of an exact zero (IEEE: -0 only when both addends are -0)."""
    if q == 0:
        return -0.0 if neg_zero else 0.0
    sign = -1.0 if q < 0 else 1.0
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()      # 2^e <= q < 2^(e+2)
    if Fraction(2) ** e > q:
        e -= 1
    if Fraction(2) ** (e + 1) <= q:
        e += 1
    quantum = Fraction(2) ** (max(e, F32_MIN_EXP) - 23)
    n = q / quantum
    fl = n.numerator // n.denominator
    rem = n - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    r = fl * quantum
    if r >= Fraction(2) ** F32_MAX_EXP:
        return sign * math.inf
    return sign * float(r)


def fma_exact(a, b, c):
    p = Fraction(a) * Fraction(b)
    neg_zero = p == 0 and c == 0 and math.copysign(1.0, a) * math.copysign(1.0, b) < 0 and math.copysign(1.0, c) < 0
    return round_f32(p + Fraction(c), neg_zero)


def f32(v):
    return struct.unpack("<f", struct.pack("<f", v))[0]


def check_fma(triples):
    a, b, c = (torch.tensor([t[i] for t in triples], dtype=torch.float32) for i in range(3))
    got = S.fma32(a, b, c)
    assert got.dtype == torch.float32
    for i, (x, y, z) in enumerate(triples):
        want = fma_exact(x, y, z)
        g = float(got[i])
        assert bits32(g) == bits32(want), ((x, y, z), g, want)


def test_fma32_random_operands():
    g = torch.Generator().manual_seed(0)
    n = 6000
    a = torch.randn(n, generator=g) * torch.exp2(torch.randint(-30, 30, (n,), generator=g).float())
    b = torch.randn(n, generator=g) * torch.exp2(torch.randint(-30, 30, (n,), generator=g).float())
    # c near a * b in magnitude (cancellation), and far above / below it (sticky bits)
    c = -(a * b) * (1.0 + torch.randn(n, generator=g) * 2.0 ** -torch.randint(1, 30, (n,), generator=g).float())
    c[: n // 3] = torch.randn(n // 3, generator=g) * torch.exp2(torch.randint(-60, 60, (n // 3,), generator=g).float())
    check_fma([(float(x), float(y), float(z)) for x, y, z in zip(a, b, c)])


def test_fma32_adversarial_operands():
    u = 2.0 ** -23
    mid = 1.0 + 2.0 ** -12                                  # mid * mid = 1 + 2^-11 + 2^-24: a tie between two fp32 values
    odd = 1.0 + 2.0 ** -12 + u                              # odd * 1 + half an ulp: a tie whose lower neighbour is odd
    fmax = f32(3.4028234663852886e38)
    cases = [
        (mid, mid, 0.0),                                    # exact midpoint, ties to the even lower value
        (mid, mid, 2.0 ** -60),                             # sticky bit above the midpoint: up (float64 rounding: down)
        (mid, mid, -2.0 ** -60),                            # sticky bit below the midpoint: down
        (odd, 1.0, 2.0 ** -24),                             # midpoint with an odd lower neighbour: up
        (odd, 1.0, 2.0 ** -24 - 2.0 ** -70),                # just below it: down
        (-mid, mid, -2.0 ** -60),                           # the negative mirror
        (3.0, 5.0, -15.0),                                  # total cancellation: +0
        (1.0 + u, 1.0 - u, -1.0),                           # (1 - 2^-46) - 1: an exact tiny result
        (2.0 ** -75, 2.0 ** -75, 0.0),                      # 2^-150: half the smallest subnormal, ties to 0
        (2.0 ** -75, 2.0 ** -75, 2.0 ** -149),              # 1.5 x 2^-149: ties to 2 x 2^-149
        (1.5 * 2.0 ** -70, 2.0 ** -70, 2.0 ** -140),        # a subnormal result with low bits to round
        (2.0 ** -64, 2.0 ** -64, -2.0 ** -126),             # cancels into the subnormal range
        (-0.0, 1.0, -0.0),                                  # -0 + -0 = -0
        (0.0, -1.0, 0.0),                                   # -0 + +0 = +0
        (-0.0, 1.0, 0.0),
        (2.0, 3.0, -6.0),                                   # exact zero from non-zero operands: +0
        (-2.0, 3.0, 6.0),
        (2.0 ** 127, 2.0, 0.0),                             # overflow to +inf
        (-(2.0 ** 127), 2.0, 0.0),                          # and -inf
        (fmax, 1.0, 2.0 ** 103),                            # the tie between the largest value and 2^128: inf
        (fmax, 1.0, 2.0 ** 103 - 2.0 ** 80),                # just below it: the largest value
        (fmax, -1.0, -(2.0 ** 104)),                        # -inf
    ]
    check_fma([(f32(a), f32(b), f32(c)) for a, b, c in cases])
    got = S.fma32(torch.tensor([-0.0, 0.0]), torch.tensor([1.0, -1.0]), torch.tensor([-0.0, 0.0]))
    assert math.copysign(1.0, float(got[0])) < 0 and math.copysign(1.0, float(got[1])) > 0
    # the midpoint case really is one the float64 shortcut gets wrong
    a, c = torch.tensor([mid]), torch.tensor([2.0 ** -60])
    assert float((a.double() * a.double() + c.double()).float()) != float(S.fma32(a, a, c))


def python_conv(x, w, scale, shift, res, k, pad_lo, relu, storage):
    """The kernel's order in exact arithmetic: per output, fmaf over (tap, channel < Cin), then * scale, + shift,
    + residual, ReLU, each rounded to fp32, then the store."""
    N, T, H, W, Cin = x.shape
    Cout = w.shape[0]
    OT, OH, OW = T, H, W
    out = []
    taps = [(a, b, c) for a in range(k[0]) for b in range(k[1]) for c in range(k[2])]
    for m in range(N * OT * OH * OW):
        ow, r = m % OW, m // OW
        oh, r = r % OH, r // OH
        ot, n = r % OT, r // OT
        row = []
        for co in range(Cout):
            acc = 0.0
            for j, (kt, kh, kw) in enumerate(taps):
                it, ih, iw = ot + kt - pad_lo[0], oh + kh - pad_lo[1], ow + kw - pad_lo[2]
                inside = 0 <= it < T and 0 <= ih < H and 0 <= iw < W
                for c in range(Cin):
                    xv = float(x[n, it, ih, iw, c]) if inside else 0.0
                    acc = fma_exact(xv, float(w[co, j, c]), acc)
            v = acc
            if scale is not None:
                v = round_f32(Fraction(v) * Fraction(float(scale[co])))
            if shift is not None:
                v = round_f32(Fraction(v) + Fraction(float(shift[co])))
            if res is not None:
                v = round_f32(Fraction(v) + Fraction(float(res[n, ot, oh, ow, co])))
            if relu:
                v = max(v, 0.0)
            row.append(v)
        out.append(row)
    return torch.tensor(out, dtype=torch.float32).to(storage)


@pytest.mark.parametrize("storage", [torch.float32, torch.float16])
def test_simt_conv_replay_matches_python_loop(storage):
    g = torch.Generator().manual_seed(5)
    N, T, H, W, Cin, Cout, k = 2, 1, 1, 3, 20, 3, (1, 1, 2)     # W-taps 2 over W = 3: the last output reads one padded tap
    pad_lo = (0, 0, 0)                                           # TF-SAME for k = 2, s = 1: nothing below, one above
    x = torch.randn(N, T, H, W, Cin, generator=g).to(storage)
    w = torch.zeros(Cout, 2, 24, dtype=storage)                  # packed with w_ld > Cin: columns past Cin are not read
    w[:, :, :Cin] = torch.randn(Cout, 2, Cin, generator=g).to(storage)
    w[:, :, Cin:] = 1e4
    scale = torch.rand(Cout, generator=g) + 0.5
    shift = torch.randn(Cout, generator=g)
    res = torch.randn(N, T, H, W, Cout, generator=g).to(storage)
    for sc, sh, rs, relu in ((scale, shift, res, True), (None, shift, None, False), (scale, None, res, False)):
        want = python_conv(x.float(), w.float(), sc, sh, rs.float() if rs is not None else None, k, pad_lo, relu, storage)
        got = S.simt_conv_replay(x, w, sc, sh, rs, k, (1, 1, 1), pad_lo, (T, H, W), relu, dtype=storage)
        assert torch.equal(got, want), (sc is None, sh is None, rs is None, relu)
        rows = torch.tensor([5, 0, 3])
        assert torch.equal(S.simt_conv_replay(x, w, sc, sh, rs, k, (1, 1, 1), pad_lo, (T, H, W), relu, rows=rows,
                                              dtype=storage), want[rows])


def test_mean_mid_replay_is_index_order_sum_then_division():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 5, 2, 4, generator=g) * torch.exp2(torch.randint(-20, 20, (3, 5, 2, 4), generator=g).float())
    got = S.mean_mid_replay(x)
    for a in range(3):
        for p in range(2):
            for c in range(4):
                s = 0.0
                for b in range(5):
                    s = round_f32(Fraction(s) + Fraction(float(x[a, b, p, c])))
                assert bits32(float(got[a, p * 4 + c])) == bits32(round_f32(Fraction(s) / 5))


OBJ = os.path.join(ROOT, "step_b200", "_obj", "conv_simt.o")
F32_SYMBOL = "_ZN4step18conv3d_simt_kernelIfEEv16step_conv_params"


def test_simt_fp32_epilogue_is_not_contracted():
    """The fp32 instance's epilogue in the built object: per output of the 4 x 4 micro-tile a predicated FMUL (scale),
    FADD (shift), FADD (residual), FMNMX with RZ (ReLU), then the store; the main loop's 16 x 16 FFMA are unpredicated."""
    tool = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump" if os.path.exists("/usr/local/cuda/bin/cuobjdump") else None)
    if tool is None or not os.path.exists(OBJ):
        pytest.skip("needs cuobjdump and the built step_b200/_obj/conv_simt.o")
    sass = subprocess.run([tool, "-sass", "-fun", F32_SYMBOL, OBJ], capture_output=True, text=True, check=True).stdout
    ops = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(@!?U?P\d\s+)?([A-Z][A-Z0-9]*)(?:\.[A-Z0-9.]+)?\s+([^;]*);", sass)
    assert len(ops) > 100, "cuobjdump printed no SASS for %s" % F32_SYMBOL
    seq = " ".join(("p" if pred else "") + op for pred, op, _ in ops)
    epilogues = re.findall(r"pFMUL (?:\S+ )*?pFADD (?:\S+ )*?pFADD (?:\S+ )*?pFMNMX (?:\S+ )*?STG", seq)
    assert len(epilogues) == 16, ("conv3d_simt_kernel<float>'s epilogue is no longer FMUL, FADD, FADD, FMNMX per output: "
                                  "tests/_simt_replay.py rounds those four operations separately", len(epilogues))
    assert all("FFMA" not in e for e in epilogues), "an FFMA inside the epilogue: scale and shift were contracted"
    assert "pFFMA" not in seq, "a predicated FFMA: the epilogue was contracted"
    assert seq.split().count("FFMA") == 256, "the main loop is no longer 16 x 16 fmaf per 16-channel block"
