"""Superresolution.folded_weights is differentiable under grad (the native SR backward's gradients reach the checkpoint's parameters
through it) and gives the same matrices with and without grad, so the packed bytes stay as they are."""
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.superres import Superresolution


def _net():
    net = Superresolution(channels=3)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(scn.synthetic_sr_state(shapes, seed=3), strict=False)
    return net


def _flat(fw):
    return [fw["conv_in_w"], fw["conv0_w"], fw["up_w"], fw["conv1_w"], *fw["bias"], *fw["rgb_w"], *fw["rgb_b"]]


def test_fold_is_differentiable_and_unchanged_by_grad_mode():
    net = _net()
    with torch.no_grad():
        ref = _flat(net.folded_weights())
    got = _flat(net.folded_weights())
    assert all(torch.equal(a, b.detach()) for a, b in zip(ref, got))
    assert all(t.requires_grad for t in got) and not any(t.requires_grad for t in ref)
    params = list(net.parameters())
    assert not any(t is p for t in got + ref for p in params)   # moving the model later leaves the fold where it is
    sum((t * torch.linspace(-1, 1, t.numel()).view(t.shape)).sum() for t in got).backward()
    params = dict(net.named_parameters())
    for name, p in params.items():
        if name.endswith("noise_strength"):
            assert p.grad is None, name                   # the strengths enter the SR head directly, not through the fold
        else:
            assert p.grad is not None and float(p.grad.abs().sum()) > 0, name


def test_fold_matches_autograd_of_the_torch_forward_direction():
    """A directional derivative of the folded up-sampling matrix against a central difference in float64."""
    net = _net().double()
    p = net.block1.conv0.weight
    d = torch.randn_like(p)
    up = net.folded_weights(torch.float64)["up_w"]
    (g,) = torch.autograd.grad((up * up).sum(), p)
    eps = 1e-6
    with torch.no_grad():
        p += eps * d
        hi = (net.folded_weights(torch.float64)["up_w"] ** 2).sum()
        p -= 2 * eps * d
        lo = (net.folded_weights(torch.float64)["up_w"] ** 2).sum()
        p += eps * d
    fd = float((hi - lo) / (2 * eps))
    assert abs(float((g * d).sum()) - fd) <= 1e-6 * max(1.0, abs(fd))
