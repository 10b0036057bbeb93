"""Host-only checks of the operand helpers of tests/test_tc_tf32_kernel.py: tf32_exact, the exactness precondition
(is_tf32) and the grid inputs whose row-kernel combinations must stay tf32-representable."""
import torch

from tests.test_tc_tf32_kernel import grid, is_tf32, tf32_exact


def test_tf32_exact_clears_the_low_mantissa_bits():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(4096, generator=g) * 10.0 ** torch.randint(-6, 6, (4096,), generator=g)
    t = tf32_exact(x)
    assert bool(((t.view(torch.int32) & 0x1FFF) == 0).all())
    assert torch.equal(tf32_exact(t), t)                                   # idempotent
    rel = ((t.double() - x.double()).abs() / x.double().abs()).max().item()
    assert rel < 2.0 ** -10                                                # truncation: below one tf32 ulp
    assert bool((t.abs() <= x.abs()).all()) and bool((torch.sign(t) == torch.sign(x)).all())
    assert torch.equal(tf32_exact(torch.tensor([0.0, -0.0, 1.0, -2.5])), torch.tensor([0.0, -0.0, 1.0, -2.5]))


def test_is_tf32_accepts_tf32_values_only():
    assert is_tf32(torch.tensor([0.0, 1.0, -3.0, 1.0 + 2.0 ** -10, 2.0 ** -100]))
    assert not is_tf32(torch.tensor([1.0 + 2.0 ** -11]))                   # an fp32 value below tf32 resolution
    assert not is_tf32(torch.tensor([1.0 + 2.0 ** -30], dtype=torch.float64))   # not even an fp32 value
    assert is_tf32(torch.tensor([1.0 + 2.0 ** -10], dtype=torch.float64))
    g = torch.Generator().manual_seed(1)
    assert not is_tf32(torch.randn(1000, generator=g))
    assert is_tf32(tf32_exact(torch.randn(1000, generator=g)).double())


def test_grid_operands_stay_exact_through_the_row_kernels():
    """The combinations the backward row kernels form before a GEMM, restated in fp64 on grid inputs: dpre (sum of
    two gradients, ReLU / dropout mask, scale 2), the discriminator's dH = (g W2) * mask and the relation
    discriminators' dHid (two products each), the TRN's dz (a masked copy)."""
    g = torch.Generator().manual_seed(2)
    a, b = grid((512, 64), 6, g).double(), grid((512, 64), 6, g).double()
    feat = grid((512, 64), 4, g, relu=True).double()
    assert bool((feat == 0).any()) and bool((a == 0).any())               # ties at 0 for the masks
    assert is_tf32((a + b) * (feat > 0) * 2.0)
    gl, W2 = grid((512, 2), 5, g).double(), grid((2, 64), 5, g).double()
    assert is_tf32((gl @ W2) * (feat > 0))
    assert is_tf32(gl[:, 0:1] * W2[0] + gl[:, 1:2] * W2[1])
    assert is_tf32(a * (feat > 0))
    # three terms would no longer fit in 11 significant bits: the precondition notices
    g3 = grid((4096, 3), 0, g).double()
    w3 = grid((3, 8), 0, g).double()
    assert not is_tf32(g3 @ w3 + 0.5 ** 12)
