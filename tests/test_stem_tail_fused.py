"""The fused ResNet stem tail (``bn_forward_presummed(..., pool=True)`` / ``bn_backward(..., pool_arg=...)``: BatchNorm + ReLU +
3x3/s2/p1 max-pool in one forward kernel and a two-pass backward from the pooled gradient) against the unfused chain
``bn_forward_presummed`` → ``maxpool_forward`` → ``maxpool_backward`` → ``bn_backward``, bit for bit: pooled output, running
statistics, mean / rstd, dx, dγ and dβ.  The taps equal the pool's except that a window whose maximum is not > 0 stores 255.

On the CPU the real bindings run over the emulated kernels (``tests/_cuda_emu.py``); the GPU tests repeat the comparison on the
device at ResNet-18's stem shape."""
import contextlib
import types

import numpy as np
import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200 import models
from pytorch_ps_mpi_b200.models import resnet as resnet_mod
from pytorch_ps_mpi_b200.ops.batchnorm import FusedBatchNormAct2d
from pytorch_ps_mpi_b200.ops.pooling import FusedMaxPool2d
from tests import _cuda_emu
from tests import test_model_integration_emulation as MI
from tests import test_multirank_engine_emulation as H
from tests.test_model_integration_emulation import world  # noqa: F401  (fixture)


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32 if t.element_size() == 4 else torch.uint8)


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _inputs(N, C, H, W, seed, dev="cpu"):
    """Stem output x with ties (a few quantised levels on half the channels), -0, a pixel that is the maximum of four
    windows; γ with negative entries; β strongly negative on one channel (every window ≤ 0 after ReLU) and -0 on another,
    whose mean is exactly 0; a pooled gradient with ties and -0."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, C, H, W, generator=g)
    x[:, ::2] = torch.randint(-6, 7, (N, (C + 1) // 2, H, W), generator=g).float() * 0.25
    x[:, 1, ::3, ::2] = -0.0
    gamma = torch.randn(C, generator=g).abs() + 0.5
    gamma[1::3] *= -1
    beta = torch.randn(C, generator=g) * 0.5
    beta[3 % C] = -20.0
    beta[2] = -0.0
    x[:, :, 3, 3] = 4.0 * torch.sign(gamma).view(1, C)                 # (3, 3) is the maximum of windows (1..2, 1..2)
    x = x.bfloat16()
    xf = x.float()
    sums = torch.cat([xf.sum((0, 2, 3)), (xf * xf).sum((0, 2, 3))])
    sums[2] = 0.0
    dp = torch.randint(-4, 5, (N, C, H // 2, W // 2), generator=g).float() * 0.5
    dp[:, :, ::2, 1::3] = torch.randn(N, C, (H // 2 + 1) // 2, len(range(1, W // 2, 3)), generator=g)
    dp[:, 0, 0, 0] = -0.0
    return (_cl(x).to(dev), gamma.bfloat16().to(dev), beta.bfloat16().to(dev), sums.to(dev), _cl(dp.bfloat16()).to(dev))


def _routes(arg, H, W):
    """Per input pixel and channel: how many windows route their gradient to it (taps 0..8; 255 routes nothing)."""
    a = arg.permute(0, 2, 3, 1).cpu().numpy().astype(np.int64)        # N, OH, OW, C
    N, OH, OW, C = a.shape
    cnt = np.zeros((N, H + 2, W + 2, C), np.int64)
    oh, ow = np.meshgrid(np.arange(OH), np.arange(OW), indexing="ij")
    for n in range(N):
        for c in range(C):
            t = a[n, :, :, c]
            ok = t != 255
            np.add.at(cnt[n, :, :, c], ((2 * oh + t // 3)[ok], (2 * ow + t % 3)[ok]), 1)   # +1 border offset
    return cnt[:, 1:H + 1, 1:W + 1]


def _compare(m, x, gamma, beta, sums, dp, eps=1e-5, mom=0.1):
    N, C, H, W = x.shape
    dev = x.device
    rm0, rv0 = torch.randn(C, device=dev) * 0.1, torch.rand(C, device=dev) + 0.5
    rm_u, rv_u, rm_f, rv_f = rm0.clone(), rv0.clone(), rm0.clone(), rv0.clone()

    c0 = m.launch_count()
    y, mean_u, rstd_u, mask = m.bn_forward_presummed(x, None, gamma, beta, rm_u, rv_u, eps, mom, True, sums)
    pooled_u, arg_u = m.maxpool_forward(y)
    c1 = m.launch_count()
    pooled_f, mean_f, rstd_f, arg_f = m.bn_forward_presummed(x, None, gamma, beta, rm_f, rv_f, eps, mom, True, sums, pool=True)
    c2 = m.launch_count()
    assert (c1 - c0, c2 - c1) == (3, 2)
    assert pooled_f.is_contiguous(memory_format=torch.channels_last) and arg_f.is_contiguous(memory_format=torch.channels_last)
    for a, b in ((pooled_f, pooled_u), (mean_f, mean_u), (rstd_f, rstd_u), (rm_f, rm_u), (rv_f, rv_u)):
        assert _same(a, b)
    want_arg = torch.where(pooled_u.float() > 0, arg_u, torch.full_like(arg_u, 255))
    assert torch.equal(arg_f, want_arg)

    dy_u = m.maxpool_backward(dp, arg_u, H, W)
    dx_u, _, dg_u, db_u = m.bn_backward(dy_u, x, mask, gamma, mean_u, rstd_u, True, False)
    c3 = m.launch_count()
    dg_f, db_f = torch.full_like(gamma, float("nan")), torch.full_like(gamma, float("nan"))
    dx_f, dres, dg_o, db_o = m.bn_backward(dp, x, x, gamma, mean_f, rstd_f, True, False, dg_f, db_f, pool_arg=arg_f)
    c4 = m.launch_count()
    assert (c3 - c2, c4 - c3) == (4, 3)
    assert dres is None and dg_o.data_ptr() == dg_f.data_ptr() and db_o.data_ptr() == db_f.data_ptr()
    for a, b in ((dx_f, dx_u), (dg_f, dg_u), (db_f, db_u)):
        assert _same(a, b)
    return arg_u, pooled_u


# ---- CPU: the real bindings over the emulated kernels -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    m = _cuda_emu.build_extension()
    if m is None:
        pytest.skip("no g++")
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield m
    m.emu.emu_set_sm_count(132)
    torch.set_num_threads(n)


@pytest.mark.parametrize("sms", [1, 3, 132])
@pytest.mark.parametrize("N,C", [(1, 8), (2, 8), (1, 64), (2, 64)])
@pytest.mark.parametrize("H,W", [(8, 8), (16, 12), (32, 32)])
def test_fused_tail_matches_the_unfused_chain_emulated(emu, sms, N, C, H, W):
    """1 or 3 SMs: the launchers' grid caps bind, so every grid-stride loop runs several times per CTA and the reduce's
    per-CTA pixel ranges span rows and images."""
    emu.emu.emu_set_sm_count(sms)
    x, gamma, beta, sums, dp = _inputs(N, C, H, W, seed=N * 1000 + C * 10 + H + W)
    arg_u, pooled_u = _compare(emu, x, gamma, beta, sums, dp)
    routes = set(np.unique(_routes(arg_u, H, W)).tolist())
    assert {0, 1, 2, 4} <= routes, routes                               # argmax of 0, 1, 2 and 4 windows
    assert bool((pooled_u[:, 3 % C] == 0).all())                        # β = -20: every window of that channel is ≤ 0


@pytest.mark.parametrize("H,W", [(9, 8), (8, 7)])
def test_odd_sizes_are_refused_and_the_model_keeps_the_unfused_chain(emu, H, W):
    x, gamma, beta, sums, _ = _inputs(1, 8, H + H % 2, W + W % 2, seed=3)
    x = _cl(x[:, :, :H, :W])
    rm, rv = torch.zeros(8), torch.ones(8)
    with pytest.raises(RuntimeError, match="even"):
        emu.bn_forward_presummed(x, None, gamma, beta, rm, rv, 1e-5, 0.1, True, sums, pool=True)
    tail = types.SimpleNamespace(bn1=FusedBatchNormAct2d(8, relu=True).bfloat16(), maxpool=FusedMaxPool2d(3, 2, 1))
    with _patched(emu):
        assert tail.bn1.maxpool_ok(_cl(torch.zeros(1, 8, 8, 8, dtype=torch.bfloat16))) and not tail.bn1.maxpool_ok(x)
        c0 = emu.launch_count()
        out = resnet_mod.ResNet._tail(tail, x, sums)
        assert emu.launch_count() - c0 == 3                              # finalize + apply, then the pool
    y = emu.bn_forward_presummed(x, None, tail.bn1.weight, tail.bn1.bias, torch.zeros(8), torch.ones(8), 1e-5, 0.1, True, sums)[0]
    assert _same(out, emu.maxpool_forward(y)[0])


@contextlib.contextmanager
def _patched(m):
    from pytorch_ps_mpi_b200.ops import ext as ops_ext
    mp = pytest.MonkeyPatch()
    mp.setattr(ops_ext, "cuda", lambda: m)
    mp.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    try:
        yield
    finally:
        mp.undo()


def _resnet18():
    torch.manual_seed(0)
    return models.resnet18(num_classes=10).to(memory_format=torch.channels_last).bfloat16()


def _batch(step):
    g = torch.Generator().manual_seed(step)
    return _cl(torch.randn(2, 3, 64, 64, generator=g).bfloat16()), torch.randint(0, 10, (2,), generator=g)


def test_resnet18_step_is_bit_identical_with_the_fused_tail(emu, monkeypatch):
    """One ResNet-18 training step at 64x64, loss and every parameter gradient, with the fused tail and without; the
    launch count tells the two paths apart (2 + 3 of our kernels instead of 3 + 4 for the tail)."""
    res = {}
    for tail in (True, False):
        monkeypatch.setattr(resnet_mod, "_FUSED_TAIL", tail)
        with _patched(emu):
            model = _resnet18()
            x, y = _batch(0)
            c0 = emu.launch_count()
            loss = torch.nn.functional.cross_entropy(model(x).float(), y)
            loss.backward()
            res[tail] = (loss.detach(), [p.grad.clone() for p in model.parameters()], emu.launch_count() - c0,
                         model.bn1.running_var.clone(), int(model.bn1.state_dict()["num_batches_tracked"]))
    a, b = res[True], res[False]
    assert _same(a[0], b[0])
    assert all(_same(p, q) for p, q in zip(a[1], b[1]))
    assert b[2] - a[2] == 2
    assert _same(a[3], b[3]) and a[4] == b[4] == 1


def test_resnet18_through_the_engine_with_the_fused_tail(world, monkeypatch):   # noqa: F811
    """Two steps through the device engine with the stem gate attached: bn1's dγ / dβ land straight in the wire arena from
    the fused backward; losses and parameters equal the unfused run's bit for bit."""
    out = {}
    for tail in (True, False):
        monkeypatch.setattr(resnet_mod, "_FUSED_TAIL", tail)
        cluster = H.Cluster(world.emu, 1)
        H._tls.world, H._tls.m = H.World(cluster, 0), MI.ModelM(cluster, world)
        with MI._lock:
            model = _resnet18()
        named = list(model.named_parameters())
        opt = ps.SGD(named, [p for _, p in named], lr=0.05, momentum=0.9, mode="ps", engine="device")
        eng = opt._engine
        model.attach(opt)
        losses = []
        for s in range(2):
            x, y = _batch(s)
            opt.zero_grad(set_to_none=True)
            loss = torch.nn.functional.cross_entropy(model(x).float(), y)
            loss.backward()
            opt.step()
            losses.append(loss.detach())
        eng.ensure_params()
        eng.check()
        out[tail] = (losses, [p.detach().clone() for p in model.parameters()], set(eng.direct_names))
        opt.close()
    a, b = out[True], out[False]
    assert {"bn1.weight", "bn1.bias"} <= a[2]
    assert all(_same(p, q) for p, q in zip(a[0], b[0]))
    assert all(_same(p, q) for p, q in zip(a[1], b[1]))


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(256, 64, 112, 112), (3, 64, 30, 46)])
def test_fused_tail_matches_the_unfused_chain_on_the_gpu(shape):
    from pytorch_ps_mpi_b200.ops import ext
    N, C, H, W = shape
    x, gamma, beta, sums, dp = _inputs(N, C, H, W, seed=7, dev="cuda")
    _compare(ext.cuda(), x, gamma, beta, sums, dp)
