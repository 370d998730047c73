"""The edge-case inputs of tests/loss_cases.py can tell a right implementation from a wrong one: each deliberately wrong numpy
variant of the Lovasz gradient / the metrics is caught by the exact comparison tests/test_losses_edges_gpu.py makes on the
kernels, on every input that is meant to catch it. Runs without a GPU."""

import numpy as np
import pytest
import torch

import loss_cases as LC
from oracle import losses_oracle

SMALL = (2, 2, 96, 96)  # 4.5 sort tiles per image


def _right(logits, targets):
    return losses_oracle.lovasz_loss(logits, targets, with_grad=True)[1]


@pytest.mark.parametrize("shape", [(1, 3, 32, 32), SMALL, (7, 2, 64, 65)])
def test_right_variant_is_the_oracle(shape):
    for name, build in list(LC.LOVASZ_TIE_CASES.items()) + [("gaussian", LC.lovasz_gaussian)]:
        if name == "tie_block" and shape[1] * shape[2] * shape[3] <= 5000:
            continue
        logits, targets = build(shape, 3)
        assert torch.equal(LC.lovasz_variant_grad(logits, targets), _right(logits, targets)), name


@pytest.mark.parametrize("name", list(LC.LOVASZ_TIE_CASES))
@pytest.mark.parametrize("order", ["scrambled", "reversed"])
def test_tie_inputs_catch_a_wrong_order_of_equal_errors(name, order):
    """(a) a sort that is not stable, (b) an ascending stable sort read backwards: both put equal errors in another order than the
    reference's, and every tie input must see that in the gradient, in every image."""
    for shape in LC.RAGGED_MULTI_TILE[:1] + [(3, 6, 32, 48)]:
        logits, targets = LC.LOVASZ_TIE_CASES[name](shape, 5)
        right, wrong = _right(logits, targets), LC.lovasz_variant_grad(logits, targets, order=order)
        for n in range(shape[0]):
            assert not torch.equal(right[n], wrong[n]), (name, order, shape, n)


def test_gaussian_logits_do_not_catch_a_wrong_order_of_equal_errors():
    """why the tie inputs exist: among the P fp32 Gaussian errors of an image (all the suite had) at most a handful of pairs are
    equal, so a wrong order of ties moves a handful of gradient elements at best, where a tie input moves thousands"""
    P = SMALL[1] * SMALL[2] * SMALL[3]
    logits, targets = LC.lovasz_gaussian(SMALL, 5)
    assert len(np.unique(LC.errors(logits, targets)[0].numpy())) > P - 10
    tied, _ = LC.lovasz_fp16_rounded(SMALL, 5)
    for order in ("scrambled", "reversed"):
        assert int((_right(logits, targets) != LC.lovasz_variant_grad(logits, targets, order=order)).sum()) < 20
        assert int((_right(tied, targets) != LC.lovasz_variant_grad(tied, targets, order=order)).sum()) > 1000


def test_one_byte_inputs_differ_in_that_byte_only():
    for byte in range(4):
        logits, targets = LC.lovasz_one_byte(SMALL, 7, byte)
        bits = LC.errors(logits, targets).view(torch.int32).numpy().view(np.uint32)
        varying = np.bitwise_or.reduce((bits ^ bits.flat[0]).ravel())
        assert varying != 0 and (varying & ~np.uint32(0xFF << (8 * byte))) == 0, (byte, hex(varying))
        assert np.isfinite(LC.errors(logits, targets).numpy()).all()
    e = LC.errors(*LC.lovasz_one_byte(SMALL, 7, 3))
    assert (e < 0).any() and (e > 0).any()  # the top byte holds the sign: both halves of the key transform


def test_tie_block_straddles_tile_boundaries():
    logits, targets = LC.lovasz_tie_block(SMALL, 5)
    for first, last in LC.tie_block_span(logits, targets):
        assert last - first + 1 >= 5000
        assert first // LC.SORT_TILE < last // LC.SORT_TILE and first % LC.SORT_TILE != 0


def test_five_values_and_subnormals_hit_the_special_errors():
    logits, targets = LC.lovasz_five_values(SMALL, 5)
    e = LC.errors(logits, targets)
    assert 0.1 < float((e == 0).float().mean()) < 0.3 and (e < 0).any()
    assert torch.all(_right(logits, targets)[e <= 0] == 0)
    logits, targets = LC.lovasz_subnormal(SMALL, 5)
    assert (logits != 0).all() and (logits.abs() < 1.2e-38).all() and torch.all(LC.errors(logits, targets) == 1)


@pytest.mark.parametrize("shape", LC.RAGGED_MULTI_TILE[:1] + [(1, 3, 32, 32), (7, 2, 64, 65)])
def test_ragged_shapes_catch_padding_counted_as_elements(shape):
    """(c) the padding of an image to whole sort tiles taking part in the cumulative sums. Only a P that is not a multiple of the
    tile can see it, which no shape of more than one tile had before."""
    logits, targets = LC.lovasz_gaussian(shape, 9)
    assert not torch.equal(_right(logits, targets), LC.lovasz_variant_grad(logits, targets, pad_first=True))
    aligned = (2, 2, 64, 64)
    logits, targets = LC.lovasz_gaussian(aligned, 9)
    assert torch.equal(_right(logits, targets), LC.lovasz_variant_grad(logits, targets, pad_first=True))


@pytest.mark.parametrize("N", [3, 5, 6, 7])
def test_batch_sizes_that_are_not_powers_of_two_catch_the_wrong_scaling(N):
    """(d) loss / N in the reference makes autograd multiply by fp32(1 / N); dividing the gradient by N differs in the last bit
    for some elements unless N is a power of two"""
    logits, targets = LC.lovasz_gaussian((N, 2, 32, 48), 11)
    assert not torch.equal(_right(logits, targets), LC.lovasz_variant_grad(logits, targets, scale="divide"))
    logits, targets = LC.lovasz_gaussian((4, 2, 32, 48), 11)
    assert torch.equal(_right(logits, targets), LC.lovasz_variant_grad(logits, targets, scale="divide"))


def test_all_equal_closed_form_is_the_oracle():
    for shape in LC.RAGGED_MULTI_TILE:
        logits, targets = LC.lovasz_all_equal(shape, 13)
        assert torch.equal(_right(logits, targets), LC.lovasz_index_order_grad(targets, shape[1]))


def test_metrics_tie_inputs_catch_the_last_maximum():
    """(e) argmax returning the last of several maximal classes"""
    for name, logits, targets in LC.metrics_tie_cases():
        right = LC.metrics_counts_variant(logits, targets)
        assert right == tuple(losses_oracle.metrics_counts(logits, targets)), name
        assert right != LC.metrics_counts_variant(logits, targets, last_max=True), name
        top = logits.max(1, keepdim=True).values
        assert float(((logits == top).sum(1) > 1).float().mean()) > 0.05, name  # ties are a real share of the pixels
        if logits.shape[1] > 2 and "zeros" not in name:  # all-zero logits always predict class 0
            t = targets.numpy()
            q = np.argmax(logits.numpy(), 1)[t > 0] / t[t > 0]
            assert ((q != 0) & (q != 1)).mean() > 0.05, name  # quotients the reference counts in no cell
    g = LC.lovasz_gaussian((3, 6, 64, 65), 1)[0]
    t = LC.targets_random(3, 6, 64, 65, 2)
    assert LC.metrics_counts_variant(g, t) == LC.metrics_counts_variant(g, t, last_max=True)  # without ties nothing is caught


def test_softmax_edge_cases_are_what_they_claim():
    cases = {c["name"]: c for c in LC.softmax_edge_cases()}
    c = cases["gaps of 80..110, maximum on the target"]
    gap = (c["logits"].max(1).values - c["logits"].min(1).values)
    e = torch.exp(-gap)  # fp32
    assert (e == 0).any() and ((e > 0) & (e < 1.17e-38)).any() and (e >= 1.17e-38).any()
    c = cases["class 2 absent from image 0"]
    assert not (c["targets"][0] == 2).any() and (c["targets"][1] == 2).any()
    for c in cases.values():  # where the float64 reference is not finite is declared, not discovered on the GPU
        x, t, w = c["logits"], c["targets"], c["weight"]
        refs = {"ce": losses_oracle.cross_entropy_loss(x, t, w), "focal": losses_oracle.focal_loss(x, t, w, gamma=2), "miou": losses_oracle.miou_loss(x, t, w)}
        assert tuple(k for k, v in refs.items() if not np.isfinite(v)) == c["undefined"], (c["name"], refs)


def test_focal_closed_form_is_the_oracle_where_autograd_is_finite():
    seen_non_finite = False
    for c in LC.softmax_edge_cases():
        if "focal" in c["undefined"]:
            continue
        x, t, w = c["logits"], c["targets"], c["weight"]
        for gamma in (0.5, 2.0, 5.0):
            loss, grad = LC.focal_reference(x, t, w, gamma)
            ref_loss, ref_grad = losses_oracle.focal_loss(x, t, w, gamma=gamma, with_grad=True)
            assert torch.isfinite(grad).all() and np.isfinite(loss), (c["name"], gamma)
            assert abs(float(loss) - float(ref_loss)) <= 1e-6 * abs(float(ref_loss)) + 1e-12, (c["name"], gamma)
            ok = torch.isfinite(ref_grad)
            assert gamma < 1 or ok.all(), (c["name"], gamma)
            seen_non_finite |= not bool(ok.all())
            pix = ok.all(1, keepdim=True).expand_as(grad)
            assert torch.allclose(grad[pix], ref_grad[pix], rtol=1e-5, atol=1e-12), (c["name"], gamma)
    assert seen_non_finite  # gamma = 0.5 on saturated pixels: why the closed form is the reference on the GPU


def test_adam_oracle_edges():
    """zero gradient with zero second moment: the denominator is eps and the parameter does not move; a saturated step count"""
    p, grads = LC.adam_inputs(1000, 3)
    zero = grads[0] == 0
    assert 50 < zero.sum() < 200
    p1, m1, v1 = losses_oracle.adam_step(p, grads[0], np.zeros_like(p), np.zeros_like(p), lr=1e-4, step=1)
    assert np.array_equal(p1[zero], p[zero]) and np.all(v1[zero] == 0) and np.isfinite(p1).all()
    p2, _, _ = losses_oracle.adam_step(p1, grads[1], m1, v1, lr=1e-4, step=100_000)
    assert np.isfinite(p2).all() and not np.array_equal(p2, p1)


def test_sort_unique_cases_are_in_contract():
    for name, keys, bits in LC.sort_unique_cases():
        assert keys.dtype == np.uint64 and LC.in_contract(keys, bits), name
    assert not LC.in_contract(np.array([5], np.uint64), 2)
