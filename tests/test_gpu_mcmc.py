"""3DGS-MCMC kernels (csrc/mcmc.cu) on the GPU: relocation against the float64 oracle (oracle/mcmc_oracle.py), and the position
noise pinned without reproducing the random numbers: on two scenes drawn with the same Philox key the normals recovered as
z = Sigma^-1 Delta / (c w), with the oracle's Sigma and w, must agree, so a mistake in Sigma, w or an activation of either scene
shows; the recovered z must be standard normal; and the update must be deterministic in the key."""
import math

import numpy as np
import pytest
import torch

from oracle import mcmc_oracle as M

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_MAX = 51
OPACITIES = (0.005, 0.1, 0.5, 0.9, 0.99, 1.0 - 2.0 ** -23)


def binoms(n_max=N_MAX):
    """The controller's table (mcmc_density_controller.py:53-60)."""
    t = torch.zeros(n_max, n_max, dtype=torch.float32)
    for n in range(n_max):
        for k in range(n + 1):
            t[n, k] = math.comb(n, k)
    return t.to(DEV)


def relocation_inputs():
    counts = list(range(1, N_MAX + 1)) + [N_MAX + 1, 77, 10 ** 6]     # above n_max: clamped
    o = torch.tensor([a for a in OPACITIES for _ in counts], dtype=torch.float32)
    N = torch.tensor([c for _ in OPACITIES for c in counts], dtype=torch.int64)
    s = torch.exp(torch.empty(o.shape[0], 3).uniform_(-7.0, 1.0, generator=torch.Generator().manual_seed(3)))
    return o, s, N


def test_relocation_matches_the_float64_oracle():
    from b200gs.mcmc import compute_relocation
    o, s, N = relocation_inputs()
    new_o, new_s = compute_relocation(o.to(DEV), s.to(DEV), N.to(DEV), binoms())
    assert new_o.shape == o.shape and new_s.shape == s.shape
    ref_o, ref_s = M.relocation(o.double().numpy(), s.double().numpy(), N.numpy(), N_MAX)
    err_o = np.abs(new_o.cpu().double().numpy() - ref_o) / ref_o
    err_s = np.abs(new_s.cpu().double().numpy() - ref_s) / ref_s
    assert err_o.max() <= 1e-6, err_o.max()
    assert err_s.max() <= 1e-5, err_s.max()


def test_relocation_int32_int64_and_gsplat_name_agree_bit_for_bit():
    from b200gs import compat
    from b200gs.mcmc import compute_relocation
    o, s, N = (t.to(DEV) for t in relocation_inputs())
    b = binoms()
    a64 = compute_relocation(o, s, N, b)
    a32 = compute_relocation(o, s, N.to(torch.int32), b)
    compat.install()
    from gsplat.relocation import compute_relocation as gsplat_compute_relocation
    ag = gsplat_compute_relocation(o, s, N, b)
    for x, y, z in zip(a64, a32, ag):
        assert torch.equal(x, y) and torch.equal(x, z)


def noise_scene(n, seed):
    """Unnormalised quaternions (norms 0.3-5), the three scales of a Gaussian within a factor 3 of each other (Sigma well
    conditioned), opacities in [0.001, 0.004] (noise weight 0.52-0.6), means 0 (the update is the noise itself)."""
    g = torch.Generator().manual_seed(seed)
    log_scales = -5.0 + 2.0 * torch.rand(n, 1, generator=g) + math.log(3.0) * torch.rand(n, 3, generator=g)
    q = torch.randn(n, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True) * (0.3 + 4.7 * torch.rand(n, 1, generator=g))
    logits = torch.logit(0.001 + 0.003 * torch.rand(n, 1, generator=g))
    return {"means": torch.zeros(n, 3), "log_scales": log_scales, "raw_quats": q, "opacity_logits": logits}


def run_noise(scene, noise_lr, xyz_lr, seed):
    from b200gs.mcmc import add_position_noise
    t = {k: v.to(DEV) for k, v in scene.items()}
    out = add_position_noise(t["means"], t["log_scales"], t["raw_quats"], t["opacity_logits"], noise_lr, xyz_lr,
                             generator=torch.Generator().manual_seed(seed))
    assert out is t["means"]
    return out.cpu()


def recover_z(scene, delta, c):
    sigma = M.covariance(scene["log_scales"].double().numpy(), scene["raw_quats"].double().numpy())
    w = M.noise_weight(scene["opacity_logits"].double().numpy())
    return np.linalg.solve(sigma, delta.double().numpy()[..., None])[..., 0] / (c * w[:, None])


def test_position_noise_arithmetic_and_distribution():
    from scipy import stats
    n, noise_lr, xyz_lr = 1_000_000, 5e5, 1.6e-4
    c = float(np.float32(noise_lr * xyz_lr))       # the kernel's scale argument is fp32
    zs = []
    for scene_seed in (1, 2):
        scene = noise_scene(n, scene_seed)
        zs.append(recover_z(scene, run_noise(scene, noise_lr, xyz_lr, seed=11), c))
    z1, z2 = zs
    rel = np.linalg.norm(z1 - z2, axis=1) / np.linalg.norm(z1, axis=1)
    assert rel.max() <= 1e-4, rel.max()
    x = z1.reshape(-1)
    m = x.size
    assert abs(x.mean()) < 5.0 / math.sqrt(m), x.mean()
    assert abs(x.var() - 1.0) < 0.01, x.var()
    assert stats.kstest(x, "norm").pvalue > 1e-3
    corr = np.corrcoef(z1.T)
    assert np.abs(corr[np.triu_indices(3, 1)]).max() < 0.01, corr


def test_position_noise_determinism_and_edges():
    from b200gs.mcmc import add_position_noise
    scene = noise_scene(4096, 5)
    scene["means"] = torch.randn(4096, 3, generator=torch.Generator().manual_seed(6))
    a, b, d = (run_noise(scene, 5e5, 1.6e-4, seed) for seed in (7, 7, 8))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert not torch.equal(a, d) and not torch.equal(a, scene["means"])
    same = run_noise(scene, 0.0, 1.6e-4, 7)
    assert torch.equal(same.view(torch.int32), scene["means"].view(torch.int32))

    # opaque Gaussians: w = 1 / (1 + e^89.5) or less, so they do not move
    opaque = noise_scene(4096, 9)
    opaque["opacity_logits"] = torch.logit(torch.empty(4096, 1).uniform_(0.9, 0.999, generator=torch.Generator().manual_seed(10)))
    opaque["log_scales"] = opaque["log_scales"] + 4.0
    assert run_noise(opaque, 5e5, 1e-2, 7).abs().max() < 1e-30

    # the key comes from torch's default generator: manual_seed reproduces a sequence of calls, and the calls of it differ
    def two_calls():
        torch.manual_seed(1234)
        t = {k: v.to(DEV) for k, v in scene.items()}
        first = add_position_noise(t["means"], t["log_scales"], t["raw_quats"], t["opacity_logits"], 5e5, 1.6e-4).cpu()
        add_position_noise(t["means"], t["log_scales"], t["raw_quats"], t["opacity_logits"], 5e5, 1.6e-4)
        return first, t["means"].cpu()
    (f1, s1), (f2, s2) = two_calls(), two_calls()
    assert torch.equal(f1, f2) and torch.equal(s1, s2)
    assert not torch.equal(f1 - scene["means"], s1 - f1)
