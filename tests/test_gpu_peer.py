"""Single-GPU test of the fused reduce-scatter -> Adam -> all-gather kernel (csrc/peer.cu, dist.PeerReduceAdam) and of the
symmetric-memory statistics exchange (dist.PeerStats) in a 1-rank process group: the kernels then read / write their "peers"
through the same pointer tables and must reproduce nl_adam_bf16_ctl and nl_stats_unpack exactly.  The W > 1 behaviour (NVLS
multicast, bit-identity with NCCL all-reduce + Adam, identical replicas) is checked by scripts/test_peer.py under torchrun
and by bench.py's strong-scaling block on every multi-GPU run."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pg():
    import torch.distributed as dist
    if dist.is_initialized():
        yield dist.group.WORLD
        return
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    yield dist.group.WORLD
    dist.destroy_process_group()


def test_peer_reduce_adam_equals_adam_kernel(pg):
    import nerfloam_b200 as nl
    cap = nl._capi
    dev = torch.device("cuda", 0)
    V, F = 3001, 2
    try:
        peer = nl.dist.PeerReduceAdam(pg, dev, V, F, lr=0.01)
    except Exception as exc:      # no symmetric-memory support on this system
        pytest.skip(f"symmetric memory unavailable: {exc!r}")
    torch.manual_seed(0)
    p0 = (torch.randn(V, 16, device=dev) * 0.01).to(torch.bfloat16)
    peer.param.copy_(p0)
    ctl = torch.zeros(cap.CTL_WORDS, dtype=torch.int32, device=dev)
    p_ref = p0.clone()
    g_ref = torch.zeros(V, 16, device=dev)
    opt = nl.engine.FusedAdam([dict(param=p_ref, grad=g_ref, lr=0.01)], ctl=ctl)
    stats = torch.zeros(nl.engine.STATS_BYTES, dtype=torch.uint8, device=dev)
    for step in (1, 2, 3):
        g = torch.randn(V, 16, device=dev) * 0.1
        g[::4] = 0
        ctl[cap.CTL_ADAM_STEP] = step
        ctl[cap.CTL_SKIP_NOW] = 1 if step == 2 else 0            # a skipped iteration must leave table and moments alone
        peer.grad.zero_()
        peer.grad[peer.n_hdr:].view(V, 16).copy_(g)
        peer.grad[16:16 + F * 12] = torch.arange(F * 12, device=dev, dtype=torch.float32)
        stats.view(torch.float64)[16:18] = torch.tensor([3.25, 1e-3 + 1e-11], dtype=torch.float64, device=dev)
        pose = torch.zeros(F, 12, device=dev)
        peer.step(stats, ctl, pose)
        g_ref.copy_(g)
        opt.step()
        torch.cuda.synchronize()
        assert torch.equal(peer.param, p_ref), step
        assert torch.equal(pose.view(-1), torch.arange(F * 12, device=dev, dtype=torch.float32))
        s = stats.view(torch.float64)[16:18].tolist()
        assert s[0] == 3.25 and abs(s[1] - (1e-3 + 1e-11)) < 1e-15
    assert torch.equal(peer.m, opt.groups[0]["m"]) and torch.equal(peer.v, opt.groups[0]["v"])


def test_peer_stats_exchange_equals_unpack(pg):
    import nerfloam_b200 as nl
    cap = nl._capi
    dev = torch.device("cuda", 0)
    try:
        ps = nl.dist.PeerStats(pg, dev)
    except Exception as exc:
        pytest.skip(f"symmetric memory unavailable: {exc!r}")
    st = cap.RenderStats()
    st.n_hit_rays, st.max_samples, st.error = 4321, 29, 2
    st.cnt_fs_valid, st.cnt_sdf_valid, st.pad_fs_rays, st.pad_fs_nsamp, st.pad_sdf_rays, st.pad_sdf_nsamp = 123456, 98765, 77, 1234, 55, 999
    st.pad_sdf_d2, st.pad_sdf_d2_nsamp = 1234.5678, 98765.4321
    a = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).cuda()
    b = a.clone()
    ps.exchange(a, 1.0, 10000.0)
    buf = torch.empty(nl.dist.stats_words(1), dtype=torch.float64, device=dev)
    nl.dist.pack_stats(b, buf, 0, 1, 0)
    nl.dist.unpack_stats(b, buf, 1, 0, 1.0, 10000.0)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    out = cap.RenderStats.from_buffer_copy(a.cpu().numpy().tobytes())
    assert out.n_hit_rays == 4321 and out.max_samples == 29 and out.error == 2 and out.g_sdf > 0
