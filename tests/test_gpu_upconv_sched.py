"""GPU tests of which upsampling layers run on the fused kernel (networks.upconv_fused; run on an H100: ``pytest -m gpu``): the
layers of a 256^2 generator that get the kernel's packed weights, and the newly dispatched 8^2 layer at the benchmark's batch of 32,
exact (construction of test_gpu_upconv.py: y must equal float32(S / 64) * float32(alpha gain d) bit for bit).  At batch 32 that
layer is 256 (image, strip, N tile) units, so on an H100 every CTA walks one or two of them and the last wave is partial."""
import pytest
import torch

from tests.test_gpu_upconv import _integer_case

pytestmark = pytest.mark.gpu


def test_generator_dispatch(gf, cuda_dev):
    """Inference with TF32 convolutions: the 8^2 and 256^2 upsampling layers get the fused kernel's packed weights, 16^2 .. 128^2
    stay on the cuDNN polyphase path."""
    G = gf.Generator(resolution=256, components_num=16, latent_dim=32).to(cuda_dev).eval()
    fused = {}
    with torch.no_grad():
        for m in G.modules():
            if getattr(m, "up", False) and hasattr(m, "_conv_weights"):
                fused[m.resolution] = m._conv_weights()[3] is not None
    assert fused == {8: True, 16: False, 32: False, 64: False, 128: False, 256: True}


def test_8x8_layer_at_batch_32_exact(gf, cuda_dev):
    _integer_case(gf, cuda_dev, 32, 4, 4, 512, 512, seed=11)
