"""`Decoder` plug-in with the constructor, state_dict keys and methods of src/variations/lidar.py:80-131
(selected by `decoder: lidar` in the YAML through import_util.get_decoder).

Parameters live in ordinary nn.Linear modules (`pts_linears.{0,1}`, `sdf_out`), so deepcopy, pickling,
.cuda(), optimisers and checkpoints behave exactly like the reference module; the arithmetic of
get_values / forward on CUDA tensors is the fused sm_90a kernel (csrc/mlp.cu) behind an autograd.Function.
Supported: depth=2, skips=[], embedder='none', in_dim=16, width in {32,64,128,256} -- the shape of every
config the reference ships; anything else raises NotImplementedError at construction.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _capi
from .engine import DecoderBuffers, alloc_act, mlp_forward, mlp_train


class Same(nn.Module):
    def __init__(self, in_dim):
        super().__init__()
        self.embedding_size = in_dim

    def forward(self, x):
        return x


class _DecoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dec, *params):
        bufs = DecoderBuffers.of(dec, x.device)
        bufs.refresh_transposes()
        M = x.shape[0]
        sdf = torch.empty(M, dtype=torch.float32, device=x.device)
        mlp_forward(bufs, M, None, x, sdf)
        ctx.save_for_backward(x)
        ctx.dec = dec
        return sdf.unsqueeze(-1)

    @staticmethod
    def backward(ctx, gout):
        (x,) = ctx.saved_tensors
        dec = ctx.dec
        bufs = DecoderBuffers.of(dec, x.device)
        bufs.refresh_transposes()
        M, W = x.shape[0], bufs.width
        sdf = torch.empty(M, dtype=torch.float32, device=x.device)
        dx = torch.empty((M, 16), dtype=torch.float32, device=x.device)
        need_w = any(ctx.needs_input_grad[2:])
        act = alloc_act(W, M, x.device) if need_w else None
        g = gout.reshape(-1).contiguous().float()
        bufs.gradflat.zero_()                       # the buffers are cached per decoder (DecoderBuffers.of): start from zero ...
        mlp_train(bufs, M, None, x, sdf, dx, need_w, act, dsdf_ext=g)
        grads = [t.clone() for t in bufs.grads] if need_w else [None] * 6      # ... and hand autograd its own copies
        return (dx if ctx.needs_input_grad[0] else None, None, *grads)


class Decoder(nn.Module):
    def __init__(self, depth=8, width=258, in_dim=3, sdf_dim=128, skips=[4], multires=6, embedder="none", point_dim=3,
                 local_coord=False, **kwargs):
        super().__init__()
        if embedder != "none":
            raise NotImplementedError("only embedder='none' is supported (no shipped config uses another one)")
        if depth != 2 or list(skips) != [] or in_dim != 16 or width not in (32, 64, 128, 256):
            raise NotImplementedError("fused decoder supports depth=2, skips=[], in_dim=16, width in {32,64,128,256} "
                                      f"(got depth={depth}, skips={skips}, in_dim={in_dim}, width={width})")
        self.D, self.W, self.skips, self.point_dim = depth, width, list(skips), point_dim
        # how to rebuild this module on the other side of a hand-off (share.ShareData sends the parameters as one flat device tensor)
        self.ctor_kwargs = dict(depth=depth, width=width, in_dim=in_dim, sdf_dim=sdf_dim, skips=list(skips), multires=multires, embedder=embedder,
                                point_dim=point_dim, local_coord=local_coord)
        self.pe = Same(in_dim)
        self.pts_linears = nn.ModuleList([nn.Linear(in_dim, width)] + [nn.Linear(width, width) for _ in range(depth - 1)])
        self.sdf_out = nn.Linear(width, 1)

    def get_values(self, input):
        x = self.pe(input)
        if not x.is_cuda:
            raise RuntimeError("Decoder runs on the GPU only (no CPU fallback): move the module and its input to cuda")
        params = [self.pts_linears[0].weight, self.pts_linears[0].bias, self.pts_linears[1].weight, self.pts_linears[1].bias,
                  self.sdf_out.weight, self.sdf_out.bias]
        return _DecoderFn.apply(x.float().contiguous(), self, *params)

    def forward(self, inputs):
        return {"sdf": self.get_values(inputs)}
