"""CPU check of the fused upsampling kernel's decomposition (csrc/gf_conv.cu, upconv_blur_tc_kernel), restated in numpy: phase
positions holding T_even[r] / T_odd[r-1], the four phase accumulators fed from the two column shifts and two row shifts, strips of
16 phase columns overlapping by two, steps of 8 phase rows with the last two carried, and the fixed-order blur -- against the
oracle's modulated transposed convolution + blur (oracle/generator.py _modconv(up=2)) in float64."""
import math

import numpy as np
import pytest
import torch

from oracle import generator as og

PC, PR = 16, 8                 # phase columns per strip, phase rows per step
OC = PC - 2                    # output column pairs per strip


def fused_np(x, w, d, gain=4.0):
    """x [H, W, I] (already style-scaled), w [O, I, 3, 3], d [O] -> y [2H, 2W, O], walking strips and steps like the kernel."""
    H, W, I = x.shape
    O = w.shape[0]
    y = np.full((2 * H, 2 * W, O), np.nan)
    tap = lambda ky, kx: w[:, :, ky, kx].T                                    # [I, O]
    for st in range((W + OC - 1) // OC):
        j0 = st * OC
        carry = np.zeros((4, 2, PC, O))                                      # unused at step 0 (rows -2, -1)
        for s in range((H + 2 + PR - 1) // PR):
            i0 = s * PR

            def view(sy, sx):                                                # x[i0 + r + sy, j0 + c + sx], zero outside
                out = np.zeros((PR, PC, I))
                for r in range(PR):
                    for c in range(PC):
                        xr, xc = i0 + r + sy, j0 + c + sx
                        if 0 <= xr < H and 0 <= xc < W:
                            out[r, c] = x[xr, xc]
                return out
            v00, v0m, vm0, vmm = view(0, 0), view(0, -1), view(-1, 0), view(-1, -1)
            ee = v00 @ tap(0, 0) + v0m @ tap(0, 2) + vm0 @ tap(2, 0) + vmm @ tap(2, 2)
            eo = v0m @ tap(0, 1) + vmm @ tap(2, 1)
            oe = vm0 @ tap(1, 0) + vmm @ tap(1, 2)
            oo = vmm @ tap(1, 1)
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


@pytest.mark.parametrize("H,W", [(4, 4), (1, 1), (5, 17), (9, 30), (8, 8), (3, 29)])
def test_fused_decomposition_matches_oracle(H, W):
    B, I, O = 2, 8, 6
    g = torch.Generator().manual_seed(H * 100 + W)
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
        got = fused_np(x[b].permute(1, 2, 0).numpy() * s, w_eff, d)
        assert not np.isnan(got).any(), "an output was never written"
        np.testing.assert_allclose(got, ref[b], rtol=1e-10, atol=1e-12)
