"""NaN-guarded output buffers and bit-exact comparison, shared by the kernel tests that call the C ABI directly.

Every output a test hands to a kernel sits in the middle of a buffer filled with a quiet NaN no arithmetic produces; after the
call the test checks that the guards before and after the output are intact and that every element of the output was written.
"""
import math

import torch

GUARD = 64                       # floats of NaN guard before and after every output buffer (keeps the outputs 16-byte aligned)
GUARD_BITS = 0x7FC0DEAD          # a quiet NaN no arithmetic produces


class Guarded:
    """An fp32 output of the given shape in the middle of a NaN-filled buffer (or preloaded with `init`)."""

    def __init__(self, shape, dev, init=None):
        self.n = math.prod(shape)
        self.buf = torch.full((self.n + 2 * GUARD,), GUARD_BITS, dtype=torch.int32, device=dev)
        self.t = self.buf[GUARD:GUARD + self.n].view(torch.float32).view(shape)
        assert self.t.data_ptr() % 16 == 0
        if init is not None:
            self.t.copy_(init)

    def ptr(self):
        return self.t.data_ptr()

    def check(self, name, written=True):
        assert (self.buf[:GUARD] == GUARD_BITS).all(), f"{name}: written before the output"
        assert (self.buf[GUARD + self.n:] == GUARD_BITS).all(), f"{name}: written past the output"
        if written:
            assert not (self.buf[GUARD:GUARD + self.n] == GUARD_BITS).any(), f"{name}: elements left unwritten"
        return self.t


def assert_exact(got, want, name):
    assert got.shape == want.shape, name
    bad = got != want                                   # -inf == -inf; a NaN never equals
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {got.numel()} elements differ, first at {bad.nonzero()[0].tolist()}: "
                           f"{got[bad][0].item()} vs {want[bad][0].item()}")
