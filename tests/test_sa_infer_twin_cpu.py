"""The fp64 twin of the pre-encoder's inference kernel (tests/sa_infer_twin.py), checked without a GPU: its structure
against the module path, the plane split it restates, and the power of the bar the GPU tests hold the kernel to."""
import copy
import math

import numpy as np
import pytest
import torch

import sa_infer_twin as T

# the (c0, b, npoint, seed) cases of test_sa_infer_edges_gpu's tight-bar test
POWER_CASES = [(3, 2, 37, 1), (6, 2, 37, 2)]


def _affine64(mlp):
    return T.folded_affine(T.blocks_of(copy.deepcopy(mlp).double()))


@pytest.mark.parametrize("c0", [3, 6])
def test_twin_with_exact_weights_is_the_module_path(c0):
    """activations unrounded and unsplit, W2 and W3 as one exact plane, affine folded in fp64: the twin's layers,
    affine folding, ReLU and max placement are the module path's"""
    mlp = T.make_mlp(c0, seed=10 + c0)
    x = T.make_input(2, c0, 37, seed=c0)
    blocks = T.blocks_of(mlp)
    w1 = blocks[0][0].weight.detach().reshape(64, c0).double()
    out, _ = T.twin(x, w1, _affine64(mlp), T.weight_planes_exact(blocks[1][0].weight),
                    T.weight_planes_exact(blocks[2][0].weight), exact=True, want_cond=False)
    exp = T.module_path(blocks, x)
    assert out.shape == exp.shape == (2 * 37, 256)
    err = float((out - exp).abs().max() / exp.abs().max())
    assert err < 1e-12, err


def test_numpy_split_reproduces_fp32_and_truncates_within_2_to_minus_16():
    """over the magnitudes weights and activations take (the split of a value near the fp32 maximum overflows plane
    0, and bf16's subnormals end at 2^-133, above fp32's)"""
    g = np.random.default_rng(0)
    x = np.concatenate([
        (g.standard_normal(200_000) * np.exp2(g.integers(-40, 40, 200_000))).astype(np.float32),
        np.array([0.0, -0.0, 1.0, -1.0, 1.00390625, 1.005859375, 2.0 ** -100, 3.0e38], np.float32),
    ])
    p = T.split_planes_np(x, 3)
    assert all(pl.dtype == np.float32 for pl in p)
    # each plane is a bf16 value
    assert all(((pl.view(np.uint32) & 0xFFFF) == 0).all() for pl in p)
    three = p[0].astype(np.float64) + p[1] + p[2]
    assert np.array_equal(three, x.astype(np.float64)), "3 planes must carry every fp32 bit"
    two = p[0].astype(np.float64) + p[1]
    nz = x != 0
    worst = float((np.abs(two - x)[nz] / np.abs(x[nz].astype(np.float64))).max())
    print(f"2-plane truncation: worst {worst:.3e} relative (bound 2^-16 = {2.0 ** -16:.3e})")
    assert worst <= 2.0 ** -16
    # the module-path bar is built on this budget
    assert T.MODULE_BAR >= 2.0 ** -16 + T.TWIN_BAR


def test_numpy_bf16_rounding_is_torchs_round_to_nearest_even():
    g = np.random.default_rng(1)
    x = (g.standard_normal(100_000) * np.exp2(g.integers(-30, 30, 100_000))).astype(np.float32)
    ties = (np.arange(1, 1000, dtype=np.uint32) << 16 | 0x8000).view(np.float32)      # exactly half-way
    x = np.concatenate([x, ties, -ties])
    got = T.bf16_rn(x)
    exp = torch.from_numpy(x).to(torch.bfloat16).float().numpy()
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))
    torch_planes = T.split_planes(torch.from_numpy(x), 3)
    for a, b in zip(T.split_planes_np(x, 3), torch_planes):
        assert np.array_equal(a.view(np.uint32), b.numpy().view(np.uint32))


@pytest.mark.parametrize("c0,b,npoint,seed", POWER_CASES)
def test_every_plane_product_moves_the_output_beyond_the_twin_bar(c0, b, npoint, seed):
    """Removing any one of the kernel's 6 + 5 plane products from the twin moves some output element by more than
    TWIN_BAR x its conditioning: a kernel that drops or repeats a product cannot pass the GPU test."""
    mlp = T.make_mlp(c0, seed)
    x = T.make_input(b, c0, npoint, seed=seed)
    ops_ = T.operands(T.blocks_of(mlp), packed=False)
    full, cond = T.twin(x, *ops_)
    weakest = math.inf
    for layer, plist in (("l2", T.L2_PRODUCTS), ("l3", T.L3_PRODUCTS)):
        for i, (pa, pb) in enumerate(plist):
            cut, _ = T.twin(x, *ops_, drop=(layer, i), want_cond=False)
            moved = float(((cut - full).abs() / cond).max())
            ratio = moved / T.TWIN_BAR
            weakest = min(weakest, ratio)
            print(f"c0={c0} without {layer} {T.product_name(pa, pb)}: moves the output by "
                  f"2^{math.log2(moved):.2f} cond = {ratio:.1f} x the twin bar")
            assert moved > T.TWIN_BAR, (layer, T.product_name(pa, pb))
    # the W3 plane the kernel leaves out is visible above the twin bar as well: the twin must not hold a third one
    w1, aff, w2p, w3p = ops_
    all3, _ = T.twin(x, w1, aff, w2p, torch.cat([w3p[:1], w3p[1:2] + w3p[2:3]]), want_cond=False)
    moved = float(((all3 - full).abs() / cond).max())
    print(f"c0={c0} with W3's third plane: moves the output by {moved / T.TWIN_BAR:.1f} x the twin bar")
    assert moved > T.TWIN_BAR
