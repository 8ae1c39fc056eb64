"""CPU check of the fused upsampling kernel's shift-grouped MMA schedule (csrc/gf_conv.cu, upconv_blur_tc_kernel), restated in
numpy from the kernel's own tables (U_GTAPS, U_GNX, U_GTAP, U_GOFF, U_GROW, read from the source): per 32-channel chunk the four
activation shifts in the kernel's issue order, each shift's taps laid side by side as one B
operand, the two accumulator fragments X = [ee, eo] and Y = [oe, oo] that every wgmma writes whole or by its first half, the first
chunk's shift (-1,-1) initialising both fragments; strips of 16 phase columns overlapping by two, steps of 8 phase rows with the
last two carried, and the fixed-order blur -- against the oracle's modulated transposed convolution + blur
(oracle/generator.py _modconv(up=2)) in float64."""
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import generator as og

PC, PR = 16, 8                 # phase columns per strip, phase rows per step
OC = PC - 2                    # output column pairs per strip
BK = 32                        # input channels per chunk
SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gansformer-reproducibility-challenge_b200", "csrc",
                   "gf_conv.cu")


def _table(src, name):
    m = re.search(r"constexpr int " + name + r"(\[4\])+ = (\{.*?\});", src)
    assert m, f"{name} not found in gf_conv.cu"
    return eval(m.group(2).replace("{", "[").replace("}", "]"))


def _groups():
    """The kernel's shift groups in issue order: (row shift, column shift, taps of fragment X (ee, eo), taps of fragment Y (oe, oo)),
    tap = ky * 3 + kx; checks that the weight boxes of consecutive groups are packed in the stage in that order."""
    src = open(SRC).read()
    ntaps, nx, taps, off, row = (_table(src, n) for n in ("U_GTAPS", "U_GNX", "U_GTAP", "U_GOFF", "U_GROW"))
    # the producer loads the column-shift -1 box before group 0 and the column-shift 0 box before group 2
    assert "j0 - (g == 0)" in src and "if (g == 0 || g == 2) {" in src
    assert off == [sum(ntaps[:g]) for g in range(4)] and sum(ntaps) == 9
    return [(0 if row[g] else -1, -1 if g < 2 else 0, tuple(taps[g][:nx[g]]), tuple(taps[g][nx[g]:ntaps[g]])) for g in range(4)]


GROUPS = _groups()


def test_groups_cover_every_tap_once():
    """Each filter tap feeds exactly the phase its (ky, kx) parity and the activation shift give it."""
    seen = []
    for sy, sx, tx, ty in GROUPS:
        for frag, taps in ((0, tx), (1, ty)):
            for pos, t in enumerate(taps):
                ky, kx = divmod(t, 3)
                row_odd, col_odd = frag, pos                 # X = [ee, eo], Y = [oe, oo]
                assert ky % 2 == row_odd and kx % 2 == col_odd
                # row: T_even[m] = w[0] x[m] + w[2] x[m-1], T_odd[m-1] = w[1] x[m-1] -> shift -1 for ky in (1, 2), 0 for ky = 0
                assert sy == (0 if ky == 0 else -1) and sx == (0 if kx == 0 else -1)
                seen.append(t)
    assert sorted(seen) == list(range(9))


def test_every_wgmma_writes_a_whole_fragment_or_its_first_half():
    for _, _, tx, ty in GROUPS:
        assert len(tx) in (1, 2) and len(ty) in (0, 1, 2)     # n64 = first half, n128 = whole fragment
    assert len(GROUPS[0][2]) == 2 and len(GROUPS[0][3]) == 2  # the first group initialises both fragments whole


def grouped_np(x, w, d, gain=4.0):
    """x [H, W, I] (already style-scaled), w [O, I, 3, 3], d [O] -> y [2H, 2W, O], walking strips, steps, chunks and shift groups
    like the kernel."""
    H, W, I = x.shape
    O = w.shape[0]
    y = np.full((2 * H, 2 * W, O), np.nan)
    for st in range((W + OC - 1) // OC):
        j0 = st * OC
        carry = np.zeros((4, 2, PC, O))                                      # [ee, eo, oe, oo] rows -2, -1: unused at step 0
        for s in range((H + 2 + PR - 1) // PR):
            i0 = s * PR
            X = Y = None
            for c0 in range(0, I, BK):
                for g, (sy, sx, tx, ty) in enumerate(GROUPS):
                    a = np.zeros((PR, PC, min(BK, I - c0)))                 # TMA box view: zero outside the image
                    for r in range(PR):
                        for c in range(PC):
                            xr, xc = i0 + r + sy, j0 + c + sx
                            if 0 <= xr < H and 0 <= xc < W:
                                a[r, c] = x[xr, xc, c0:c0 + BK]
                    for taps, frag in ((tx, "X"), (ty, "Y")):
                        if not taps:
                            continue
                        b = np.concatenate([w[:, c0:c0 + BK, t // 3, t % 3] for t in taps], axis=0)   # side-by-side boxes
                        part = a @ b.T                                                               # [PR, PC, 64 * len]
                        if c0 == 0 and g == 0:
                            acc = part                                                               # scale-d 0
                        else:
                            acc = (X if frag == "X" else Y).copy()
                            acc[..., :part.shape[-1]] += part                                        # whole or first half
                        if frag == "X":
                            X = acc
                        else:
                            Y = acc
            ee, eo, oe, oo = X[..., :O], X[..., O:], Y[..., :O], Y[..., O:]
            T = np.concatenate([carry, np.stack([ee, eo, oe, oo])], axis=1)  # [phase, 10 rows, 16 cols, O]
            carry = T[:, PR:PR + 2]

            def hblur(ph_e, ph_o, r):                                        # -> [2 parities, 14 pairs, O]
                E, Od = T[ph_e, r], T[ph_o, r]
                h0 = ((Od[0:OC] + 3 * E[0:OC]) + 3 * Od[1:OC + 1]) + E[1:OC + 1]
                h1 = ((E[0:OC] + 3 * Od[1:OC + 1]) + 3 * E[1:OC + 1]) + Od[2:OC + 2]
                return np.stack([h0, h1])
            for k in range(PR):
                io = i0 - 2 + k
                if not 0 <= io < H:
                    continue
                Ho0, He0, Ho1, He1, Ho2 = hblur(2, 3, k), hblur(0, 1, k), hblur(2, 3, k + 1), hblur(0, 1, k + 1), hblur(2, 3, k + 2)
                ye = ((Ho0 + 3 * He0) + 3 * Ho1) + He1
                yo = ((He0 + 3 * Ho1) + 3 * He1) + Ho2
                n = min(OC, W - j0)
                f = gain * d / 64
                y[2 * io, 2 * j0:2 * (j0 + n)] = ye[:, :n].transpose(1, 0, 2).reshape(2 * n, O) * f
                y[2 * io + 1, 2 * j0:2 * (j0 + n)] = yo[:, :n].transpose(1, 0, 2).reshape(2 * n, O) * f
    return y


# sizes off the strip and the step, one and several chunks (I = 8, 40, 64), a 1 x 1 input
@pytest.mark.parametrize("H,W,I", [(4, 4, 8), (1, 1, 8), (5, 17, 40), (9, 30, 8), (8, 8, 64), (3, 29, 40)])
def test_grouped_schedule_matches_oracle(H, W, I):
    B, O = 2, 6
    g = torch.Generator().manual_seed(H * 100 + W + I)
    x = torch.randn(B, I, H, W, generator=g, dtype=torch.float64)
    weight = torch.randn(O, I, 3, 3, generator=g, dtype=torch.float64)
    styles = torch.rand(B, I, generator=g, dtype=torch.float64) + 0.5
    f = torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=torch.float64)
    f = torch.outer(f, f) / 64
    ref = og._modconv(x, weight, styles, demodulate=True, up=2, f=f).permute(0, 2, 3, 1).numpy()
    w_eff = weight.numpy() / math.sqrt(I * 9)
    for b in range(B):
        s = styles[b].numpy()
        d = 1.0 / np.sqrt(((w_eff * s[None, :, None, None]) ** 2).sum(axis=(1, 2, 3)) + 1e-8)
        got = grouped_np(x[b].permute(1, 2, 0).numpy() * s, w_eff, d)
        assert not np.isnan(got).any(), "an output was never written"
        np.testing.assert_allclose(got, ref[b], rtol=1e-10, atol=1e-12)
