"""The fp64 decoder yardstick (tests/decoder_ref.py) against autograd: the forward pass, d features and the six weight gradients at
every width through the oracle's decoder in float64, the in-kernel loss through a direct autograd of its masked squared errors, its
fp32 roundings through a NumPy float32 restatement, and the per-problem sums of the batched loss.  No GPU needed."""
import numpy as np
import pytest
import torch

import decoder_ref as R

WIDTHS = (32, 64, 128, 256)
TRUNC = 0.3


def rel(a, b):
    return float((a - b).norm() / b.norm())


def _decoder(W, seed):
    """A seeded nl.lidar.Decoder of width W, its fp64 copy in the oracle's restatement of the reference decoder, and R's params."""
    import nerfloam_b200 as nl
    from oracle import chain as OC
    torch.manual_seed(seed)
    dec = nl.lidar.Decoder(depth=2, width=W, in_dim=16, skips=[], embedder="none", multires=0)
    ora = OC.Decoder(depth=2, width=W, in_dim=16)
    ora.load_state_dict(dec.state_dict())
    return ora.double(), R.params64(dec)


def _inputs(M, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(M, 16, generator=gen, dtype=torch.float64) * 0.05
    g = torch.randn(M, generator=gen, dtype=torch.float64) * 0.1
    return x, g


@pytest.mark.parametrize("W", WIDTHS)
def test_forward_and_backward_equal_fp64_autograd(W, monkeypatch):
    monkeypatch.setattr(R, "CHUNK", 97)          # several chunks, the last one partial
    ora, p = _decoder(W, 40 + W)
    x, g = _inputs(300, W)
    x.requires_grad_()
    lin0, lin1 = ora.pts_linears
    z1 = lin0(x)
    z2 = lin1(torch.relu(z1))
    sdf = ora.get_values(x).reshape(-1)
    (sdf * g).sum().backward()
    got = R.forward(x.detach(), p, keep=("z1", "h1", "z2", "h2", "sdf"))
    for name, ref in (("z1", z1), ("h1", torch.relu(z1)), ("z2", z2), ("h2", torch.relu(z2)), ("sdf", sdf)):
        assert rel(got[name], ref.detach()) <= 1e-12, name
    dx, grads, a_dx = R.backward(x.detach(), g, p, with_abs=True)
    assert rel(dx, x.grad) <= 1e-12
    auto = [ora.pts_linears[0].weight, ora.pts_linears[0].bias, ora.pts_linears[1].weight, ora.pts_linears[1].bias, ora.sdf_out.weight,
            ora.sdf_out.bias]
    for i, (a, t) in enumerate(zip(grads, auto)):
        assert a.shape == t.shape and rel(a, t.grad) <= 1e-12, i
    assert bool((a_dx >= dx.abs() * (1 - 1e-12)).all())


@pytest.mark.parametrize("W", WIDTHS)
def test_absolute_evaluation_bounds_every_term(W):
    _, p = _decoder(W, 7 + W)
    x, _ = _inputs(200, W + 1)
    f = R.forward(x, p, keep=("z1", "z2", "sdf"))
    a1, a2, a_sdf = R.absolute(x, p)
    assert bool((a1 >= f["z1"].abs()).all() and (a2 >= f["z2"].abs()).all() and (a_sdf >= f["sdf"].abs()).all())
    # nonnegative inputs and parameters: the absolute evaluation is the network itself
    pa = [t.abs() for t in p]
    fa = R.forward(x.abs(), pa, keep=("z1", "z2", "sdf"))
    assert torch.equal(R.absolute(x, p)[2], fa["sdf"]) and torch.equal(a1, fa["z1"]) and torch.equal(a2, fa["z2"])


def test_near_zero_flags_rows_at_a_relu_kink():
    _, p = _decoder(64, 3)
    x, _ = _inputs(500, 4)
    near = R.near_zero(x, p)
    assert float(near.float().mean()) < 0.2
    # move a row that is not near zero onto the kink of layer-1 unit 5: z1[far, 5] = 0
    W0, b0 = p[0], p[1]
    far = (~near).nonzero()[0, 0]
    x2 = x.clone()
    z = x2[far] @ W0[5] + b0[5]
    x2[far] -= z * W0[5] / (W0[5] @ W0[5])
    assert bool(R.near_zero(x2, p)[far]) and not bool(near[far])


def _samples(M, n_rays, seed, with_cos=True):
    gen = torch.Generator().manual_seed(seed)
    ray = torch.sort(torch.randint(0, n_rays, (M,), generator=gen)).values.to(torch.int32)
    flag = torch.randint(0, 3, (M,), generator=gen).to(torch.uint8)
    gt = (2.0 + 28.0 * torch.rand(n_rays, generator=gen)).float()
    cos = (0.5 + 0.5 * torch.rand(n_rays, generator=gen)).float() if with_cos else None
    c = cos[ray.long()] if with_cos else 1.0
    depth = (gt[ray.long()] / c + 0.6 * (torch.rand(M, generator=gen) - 0.5)).float()
    sdf = (0.2 * torch.randn(M, generator=gen)).float()
    return sdf, flag, depth, ray, gt, cos


@pytest.mark.parametrize("with_cos", [True, False])
def test_loss_equals_autograd_of_the_masked_squared_errors(with_cos):
    sdf, flag, depth, ray, gt, cos = _samples(3000, 400, 1, with_cos)
    g_fs, g_sdf = 0.37 / 3000, 1e4 / 3000
    fs, sd, dsdf = R.loss(sdf.double(), flag, depth, ray, gt, cos, TRUNC, g_fs, g_sdf)
    # direct statement in fp64 with the fp32 values the kernel reads (truncation and the constants are fp32 parameters)
    t, gf, gs = (float(np.float32(v)) for v in (TRUNC, g_fs, g_sdf))
    s = sdf.double().requires_grad_()
    z = depth.double() * (cos.double()[ray.long()] if with_cos else 1.0)
    front, band = (flag & 1).bool(), (flag & 2).bool()
    e_fs = (s - 1.0)[front]
    e_sdf = ((z + s * t) - gt.double()[ray.long()])[band]
    (gf * (e_fs ** 2).sum() + gs * (e_sdf ** 2).sum()).backward()
    assert abs(fs - float((e_fs ** 2).sum().detach())) <= 1e-12 * fs
    assert abs(sd - float((e_sdf ** 2).sum().detach())) <= 1e-12 * sd
    assert rel(dsdf, s.grad) <= 1e-12
    assert bool((dsdf[flag == 0] == 0).all())


@pytest.mark.parametrize("with_cos", [True, False])
def test_loss_on_fp32_sdf_rounds_like_the_kernel(with_cos):
    """On the kernel's fp32 sdf the errors are formed in fp32, one rounding per operation (mlp.cu: __fmul_rn, __fadd_rn, __fsub_rn)."""
    sdf, flag, depth, ray, gt, cos = _samples(2000, 300, 2, with_cos)
    fs, sd, _ = R.loss(sdf, flag, depth, ray, gt, cos, TRUNC, 1.0, 1.0)
    f32 = np.float32
    s, d, r, fl = sdf.numpy(), depth.numpy(), ray.numpy(), flag.numpy()
    z = d * cos.numpy()[r] if with_cos else d
    e_sdf = (z + s * f32(TRUNC)) - gt.numpy()[r]
    e_fs = s - f32(1.0)
    assert e_sdf.dtype == np.float32 and e_fs.dtype == np.float32
    ref_fs = float(np.sum(np.where(fl & 1, e_fs.astype(np.float64) ** 2, 0.0)))
    ref_sd = float(np.sum(np.where(fl & 2, e_sdf.astype(np.float64) ** 2, 0.0)))
    assert abs(fs - ref_fs) <= 1e-14 * ref_fs and abs(sd - ref_sd) <= 1e-14 * ref_sd
    # and they differ from the fp64 sums by more than that: the fp32 roundings are what the restatement reproduces
    fs64, sd64, _ = R.loss(sdf.double(), flag, depth, ray, gt, cos, TRUNC, 1.0, 1.0)
    assert abs(sd64 - ref_sd) > 1e-12 * ref_sd


def test_per_problem_sums():
    K, RP = 5, 80
    sdf, flag, depth, ray, gt, cos = _samples(2500, K * RP, 3)
    g_fs = [0.5 / (k + 1) for k in range(K)]
    g_sdf = [1e4 * (k + 2) for k in range(K)]
    fs, sd, dsdf = R.problem_loss(sdf, flag, depth, ray, gt, cos, TRUNC, RP, g_fs, g_sdf)
    k_of = ray.long() // RP
    for k in range(K):
        sel = k_of == k
        f1, s1, d1 = R.loss(sdf[sel], flag[sel], depth[sel], ray[sel], gt, cos, TRUNC, g_fs[k], g_sdf[k])
        assert abs(float(fs[k]) - f1) <= 1e-14 * f1 and abs(float(sd[k]) - s1) <= 1e-14 * s1
        assert torch.equal(dsdf[sel], d1)
    # with equal constants the problems add up to the single-problem loss
    fs_e, sd_e, d_e = R.problem_loss(sdf, flag, depth, ray, gt, cos, TRUNC, RP, [0.25] * K, [3.0] * K)
    f_all, s_all, d_all = R.loss(sdf, flag, depth, ray, gt, cos, TRUNC, 0.25, 3.0)
    assert abs(float(fs_e.sum()) - f_all) <= 1e-13 * f_all and abs(float(sd_e.sum()) - s_all) <= 1e-13 * s_all
    assert torch.equal(d_e, d_all)


def test_rows_without_gradient_or_flag_contribute_nothing():
    _, p = _decoder(128, 5)
    x, g = _inputs(400, 6)
    off = torch.arange(400) % 3 == 0
    g[off] = 0.0
    dx, grads = R.backward(x, g, p)
    assert bool((dx[off] == 0).all())
    dx_on, grads_on = R.backward(x[~off], g[~off], p)
    assert torch.equal(dx[~off], dx_on)
    for a, b in zip(grads, grads_on):
        assert rel(a, b) <= 1e-14
    sdf, flag, depth, ray, gt, cos = _samples(1000, 200, 7)
    fs, sd, dsdf = R.loss(sdf, flag, depth, ray, gt, cos, TRUNC, 0.1, 10.0)
    on = flag != 0
    fs1, sd1, _ = R.loss(sdf[on], flag[on], depth[on], ray[on], gt, cos, TRUNC, 0.1, 10.0)
    assert bool((dsdf[~on] == 0).all())
    assert abs(fs - fs1) <= 1e-14 * fs and abs(sd - sd1) <= 1e-14 * sd
