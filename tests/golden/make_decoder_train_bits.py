"""Record tests/golden/decoder_train_bits.npz: the per-sample outputs of the tensor-core decoder training kernel (k_mlp_wg) as
SHA-256 digests, so that a rework of the kernel can be held to the exact bits it produced before.

What is recorded, per case, is everything the kernel writes per sample: sdf, d feats and, with weight gradients, the whole
activation buffer (the dh1 plane [cap][256], the relu'(h2) words [cap][8], d loss / d sdf [cap]).  Every output array is filled
with NaN before the call, so the digests also pin that nothing is written past the sample count.  None of these involve atomics,
so they are deterministic.  The loss sums (fp64 atomics) and the weight gradients (fp32 atomics) are left to the other tests.

Cases: M = 300, 16 384 (whole tiles) and 16 973 (132 * 128 + 77), with and without weight gradients, against an external
d loss / d sdf; M = 16 973 through the kernel's own loss (the sample arrays of render.npz) with and without weight gradients;
a device-side sample count below the capacity; and nl_mlp_tc_train_batch with 3 problems.  All inputs come from seeded CPU
generators.  For M = 300 the full arrays are stored as well, to diagnose a mismatch.

Run:  python tests/golden/make_decoder_train_bits.py      (needs a GPU; NL_GOLDEN_OUT=<dir> writes elsewhere)
"""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from util import golden, load_decoder  # noqa: E402

NAME = "decoder_train_bits.npz"
TRUNC = 0.3
FULL_M = 300          # cases at this size also store their full arrays


def digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def _stats(nl, g_fs, g_sdf):
    s = nl._capi.RenderStats()
    s.g_fs, s.g_sdf = g_fs, g_sdf
    return bytes(s)


def _loss_inputs(z, M, gen, n_problems=1):
    """Sample arrays for the kernel's own loss: depths and rays of render.npz tiled to M samples, seeded flags."""
    R = z["cos"].shape[0]
    depth = np.resize(z["s_depth"].reshape(-1), M).astype(np.float32)
    ray = (np.arange(M) // 14 % (R * n_problems)).astype(np.int32)
    flag = torch.randint(0, 4, (M,), generator=gen, dtype=torch.int32).to(torch.uint8)
    cos = np.tile(z["cos"], n_problems).astype(np.float32)
    gt = np.tile(np.linalg.norm(z["pts"], axis=1) * z["cos"], n_problems).astype(np.float32)
    return flag, torch.from_numpy(depth), torch.from_numpy(ray), torch.from_numpy(cos), torch.from_numpy(gt), R


def run_cases(nl):
    """{case: {array: device tensor}} from the current build."""
    E, lib, ptr = nl.engine, nl._capi.lib(), nl._capi.ptr
    dev = torch.device("cuda")
    z = golden("render.npz")
    dec = load_decoder(z, "dec_")
    bufs = E.DecoderBuffers(dec, dev)
    bufs.refresh_transposes()
    out = {}

    def train(tag, M_cap, x, wgrad, count=None, dsdf=None, loss=None):
        sdf = torch.full((M_cap,), float("nan"), device=dev)
        dx = torch.full((M_cap, 16), float("nan"), device=dev)
        act = E.alloc_act(256, M_cap, dev)
        act["buf"].fill_(float("nan"))
        mdev = torch.tensor([count], dtype=torch.int32, device=dev) if count is not None else None
        bufs.gradflat.zero_()
        kw = dict(dsdf_ext=dsdf)
        if loss is not None:
            flag, depth, ray, cos, gt, _ = loss
            st = torch.frombuffer(bytearray(_stats(nl, 1.0 / M_cap, 1e4 / M_cap)), dtype=torch.uint8).to(dev)
            kw.update(s_flag=flag.to(dev), s_depth=depth.to(dev), s_ray=ray.to(dev), cos=cos.to(dev), gt_depth=gt.to(dev),
                      stats_ptr=ptr(st), truncation=TRUNC)
        E.mlp_train(bufs, M_cap, C.c_void_p(mdev.data_ptr()) if mdev is not None else None, x, sdf, dx, wgrad, act, **kw)
        torch.cuda.synchronize()
        out[tag] = {"sdf": sdf, "dfeats": dx}
        if wgrad:
            out[tag]["act"] = act["buf"]

    for M in (FULL_M, 16_384, 132 * 128 + 77):
        gen = torch.Generator().manual_seed(M)
        x = (torch.randn(M, 16, generator=gen) * 0.1).to(dev)
        g = (torch.randn(M, generator=gen) * 0.1).to(dev)
        for wgrad in (True, False):
            train(f"ext_M{M}_wgrad{int(wgrad)}", M, x, wgrad, dsdf=g)

    M = 132 * 128 + 77
    gen = torch.Generator().manual_seed(7)
    x = (torch.randn(M, 16, generator=gen) * 0.1).to(dev)
    loss = _loss_inputs(z, M, gen)
    for wgrad in (True, False):
        train(f"loss_M{M}_wgrad{int(wgrad)}", M, x, wgrad, loss=loss)

    count = M - 128 - 45
    gen = torch.Generator().manual_seed(9)
    x = (torch.randn(M, 16, generator=gen) * 0.1)
    g = (torch.randn(M, generator=gen) * 0.1)
    x[count:], g[count:] = float("nan"), float("nan")
    train(f"count_M{M}_n{count}_wgrad1", M, x.to(dev), True, count=count, dsdf=g.to(dev))

    K = 3
    gen = torch.Generator().manual_seed(11)
    x = (torch.randn(M, 16, generator=gen) * 0.1).to(dev)
    flag, depth, ray, cos, gt, R = (t.to(dev) if torch.is_tensor(t) else t for t in _loss_inputs(z, M, gen, K))
    pst = torch.frombuffer(bytearray(b"".join(_stats(nl, 0.5 / (k + 1) / M, 1e4 / (k + 1) / M) for k in range(K))),
                           dtype=torch.uint8).to(dev)
    sdf = torch.full((M,), float("nan"), device=dev)
    dx = torch.full((M, 16), float("nan"), device=dev)
    p = bufs.params
    nl._capi.check(lib.nl_mlp_tc_train_batch(M, None, ptr(x), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]),
                                             ptr(flag), ptr(depth), ptr(ray), ptr(cos), ptr(gt), ptr(pst), R, TRUNC, ptr(sdf), ptr(dx),
                                             nl._capi.stream_ptr()), "nl_mlp_tc_train_batch")
    torch.cuda.synchronize()
    out[f"batch{K}_M{M}"] = {"sdf": sdf, "dfeats": dx}
    return out


def main():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available(), "make_decoder_train_bits.py needs a GPU"
    rec = {}
    for case, arrays in run_cases(nl).items():
        for name, t in arrays.items():
            rec[f"{case}/{name}/sha256"] = np.array(digest(t))
            if case.startswith(f"ext_M{FULL_M}_"):
                rec[f"{case}/{name}"] = t.cpu().numpy()
    path = os.path.join(os.environ.get("NL_GOLDEN_OUT", HERE), NAME)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **rec)
    print(f"wrote {path}: {sum(k.endswith('/sha256') for k in rec)} digests")


if __name__ == "__main__":
    main()
