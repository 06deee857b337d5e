"""The MODEL-SIDE Python of the package on the CPU: ``models.ResNet`` (fused stem in the GEMM arena layout, ``attach`` gate),
``ops.batchnorm`` / ``ops.pooling`` / ``ops.stem`` autograd functions with direct gradient placement, driven by 2 ranks of the real
device engine — over ``_psb200_emu``, the repository's own ``bindings.cpp`` + ``gemm_bindings.cpp`` linked against the emulated
kernels (``tests/_cuda_emu.py``: BatchNorm, max-pool, im2col, wgrad finalize and every PS kernel are the real source; the three
tensor-core entry points are ATen reference math with the same contract).

``Tensor.is_cuda`` is patched to ``True`` for the duration of a test so that the package takes its device paths with host
tensors; nothing in the package is changed for this."""
import contextlib
import threading

import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200 import models, runtime
from pytorch_ps_mpi_b200.ops import ext as ops_ext
from pytorch_ps_mpi_b200.parallel import device_engine as de
from tests import _cuda_emu
from tests import test_multirank_engine_emulation as H
from tests.test_device_engine_control_flow import FakeEvent, FakeStream


class ModelM(H.RealM):
    """+ the gated stem: the consumer's flag acquire is polled here (a spin inside the call would hold the GIL)."""

    def stem_fwd(self, x, w2d, want_sums=True, flag_ptr=0, epoch=0, timeout_s=30.0):
        if flag_ptr:
            self.cluster.poll(lambda: H._words(flag_ptr, 1)[0] >= epoch, "gated PARAMS_READY (stem)")
            self.log.append(("gate", epoch))
        return self.x.stem_fwd(x, w2d, want_sums, flag_ptr, epoch, timeout_s)


    def bcast_gemm(self, x, w_ptr, N, K, bias, relu, flag_ptr=0, epoch=0, timeout_s=30.0, variant=0):
        if flag_ptr:
            self.cluster.poll(lambda: H._words(flag_ptr, 1)[0] >= epoch, "gated PARAMS_READY (GEMM)")
            self.log.append(("gate", epoch))
        return self.x.bcast_gemm(x, w_ptr, N, K, bias, relu, flag_ptr, epoch, timeout_s, variant)


@pytest.fixture
def world(monkeypatch):
    extm = _cuda_emu.build_extension()
    if extm is None:
        pytest.skip("no g++")
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    H._EXT = extm
    H._tls.world, H._tls.m = H.World(H.Cluster(extm.emu, 1), 0), None
    monkeypatch.setattr(runtime, "world", lambda: H._tls.world)
    monkeypatch.setattr(ops_ext, "cuda", lambda: H._tls.m)
    monkeypatch.setattr(de, "SymmetricArena", H.SharedArena)
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setenv("PSB200_CHUNK_BYTES", str(2048 * 2 * 8))
    yield extm
    H._EXT = None
    torch.set_num_threads(n)


_lock = threading.Lock()


def _tiny_resnet():
    """The package's ResNet with one BasicBlock stage: stem (GEMM-layout weight) → BN+ReLU → max-pool → block → fc."""
    with _lock:
        torch.manual_seed(0)
        m = models.ResNet(models.resnet.BasicBlock, [1, 1, 1, 1], num_classes=10)
        m.layer2 = m.layer3 = m.layer4 = torch.nn.Identity()
        m.fc = torch.nn.Linear(64, 10)
        return m.to(memory_format=torch.channels_last).bfloat16()


def _batch(rank, step):
    g = torch.Generator().manual_seed(50 * rank + step)
    x = torch.randn(2, 3, 16, 16, generator=g).bfloat16().contiguous(memory_format=torch.channels_last)
    return x, torch.randint(0, 10, (2,), generator=g)


def _run(extm, n, steps, attach=True):
    cluster = H.Cluster(extm.emu, n)
    out, errs = [None] * n, []

    def main(rank):
        H._tls.world, H._tls.m = H.World(cluster, rank), ModelM(cluster, extm)
        try:
            model = _tiny_resnet()
            named = list(model.named_parameters())
            opt = ps.SGD(named, [p for _, p in named], lr=0.05, momentum=0.9, weight_decay=1e-4, mode="ps", engine="device")
            eng = opt._engine
            assert eng is not None and eng.size == n
            if attach:
                model.attach(opt)
            losses = []
            for s in range(steps):
                x, y = _batch(rank, s)
                opt.zero_grad(set_to_none=True)
                loss = torch.nn.functional.cross_entropy(model(x).float(), y)
                loss.backward()
                opt.step()
                losses.append(float(loss.detach()))
            if attach:
                eng.ensure_params()
            eng.check()
            H._tls.world.barrier()
            stem_w = model.conv1.weight
            res = dict(params=[p.detach().clone() for p in model.parameters()], losses=losses, direct=set(eng.direct_names),
                       direct_n=eng.direct_grads, stem_strides=tuple(stem_w.stride()), log=list(H._tls.m.log),
                       nbt=int(model.bn1.state_dict()["num_batches_tracked"]), rm=model.bn1.running_mean.clone())
            opt.close()
            out[rank] = res
        except BaseException as exc:       # noqa: BLE001
            errs.append(exc)
            cluster.fail(exc)

    ts = [threading.Thread(target=main, args=(r,), daemon=True) for r in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in ts), "a rank thread is stuck"
    if errs:
        real = [e for e in errs if "another rank" not in str(e) and not isinstance(e, threading.BrokenBarrierError)]
        raise (real or errs)[0]
    return out


def test_resnet_through_the_engine_direct_placement_equals_encode_path(world, monkeypatch):
    """Two ranks, three steps of the tiny ResNet with the stem gate attached.  Producers we own (BatchNorm dγ/dβ, the stem weight
    gradient in its [64,176] layout) write straight into the wire arena; with ``PSB200_DIRECT_GRAD=0`` the same gradients take the
    encode pass.  The emulated kernels are deterministic, so the two runs must agree bit for bit — and ranks must be identical,
    the stem weight must live in the GEMM layout, workers must have acquired the broadcast through the gate only."""
    steps = 3
    a = _run(world, 2, steps)
    monkeypatch.setenv("PSB200_DIRECT_GRAD", "0")
    b = _run(world, 2, steps)
    for r in range(2):
        for p, q in zip(a[r]["params"], a[0]["params"]):
            assert torch.equal(p, q)                                       # ranks identical
        for p, q in zip(a[r]["params"], b[r]["params"]):
            assert torch.equal(p, q)                                       # direct placement == encode path
        assert b[r]["direct_n"] == 0
        assert a[r]["stem_strides"] == (176, 1, 24, 3)
        assert a[r]["nbt"] == steps and float(a[r]["rm"].abs().max()) > 0  # lazy num_batches_tracked, running stats moved
        assert all(torch.isfinite(p).all() for p in a[r]["params"])
    names = a[1]["direct"]
    assert "conv1.weight" in names and {"bn1.weight", "bn1.bias", "layer1.0.bn1.weight", "layer1.0.bn2.bias"} <= names, names
    assert a[0]["direct_n"] == steps * len(names)
    # the worker never queued the plain wait kernel during training: PARAMS_READY was acquired by the stem (steps 1..), and once
    # at the end by ensure_params()
    waits = [e for e in a[1]["log"] if e[0] == "wait" and e[1] == H.M.SIG_PARAMS_READY]
    gates = [e for e in a[1]["log"] if e[0] == "gate"]
    assert len(waits) == 1 and [g[1] for g in gates] == list(range(1, steps)), (waits, gates)
    assert a[0]["losses"] != a[1]["losses"]                                # different data per rank


def test_resnet_matches_a_plain_torch_model_loosely(world):
    """Same tiny ResNet, ONE rank, one step, against stock ``torch.nn`` modules in fp32 on the same weights and data (bf16 kernels
    vs fp32 math: loose tolerance) — catches sign / layout / ordering mistakes that self-consistency checks cannot."""
    res = _run(world, 1, 1, attach=False)[0]
    ref = _tiny_resnet().float()

    class Plain(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, x):
            m = self.m
            bn = lambda b, t: torch.nn.functional.batch_norm(t, None, None, b.weight, b.bias, True, 0.1, b.eps)      # noqa: E731
            x = torch.nn.functional.max_pool2d(torch.relu(bn(m.bn1, m.conv1(x))), 3, 2, 1)
            blk = m.layer1[0]
            out = torch.relu(bn(blk.bn1, blk.conv1(x)))
            out = torch.relu(bn(blk.bn2, blk.conv2(out)) + x)
            return m.fc(torch.flatten(m.avgpool(out), 1))

    plain = Plain(ref)
    o = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    x, y = _batch(0, 0)
    before = [p.detach().clone() for p in ref.parameters()]
    torch.nn.functional.cross_entropy(plain(x.float()), y).backward()
    o.step()
    for (name, _), got, want, b0 in zip(ref.named_parameters(), res["params"], ref.parameters(), before):
        step = (want.detach() - b0)
        err = (got.float() - want.detach()).abs().max()
        # the update itself (≈ lr·grad) must be reproduced to bf16 accuracy; parameters are stored in bf16 (2^-8 relative)
        assert float(err) <= 0.1 * float(step.abs().max()) + 2.0 ** -7 * float(want.detach().abs().max()) + 1e-3, (name, float(err))


@pytest.mark.parametrize("pull", [False, True])
def test_gated_first_linear_of_an_mlp(world, pull):
    """``convert_first_linear`` + ``BcastLinear.attach``: the first forward GEMM acquires the broadcast epoch itself (no wait kernel
    on workers), optionally reading the weight from the SERVER's arena (``pull``), and writes dW straight into the wire arena — 3
    ranks, bf16 parameters with fp32 masters, against the grad-gather oracle (each step: every rank's actual gradients, summed in
    fp32, reference SGD on fp32 shadows)."""
    from pytorch_ps_mpi_b200.ops.linear import BcastLinear, convert_first_linear
    n, steps = 3, 3
    hyper = dict(lr=0.05, momentum=0.9)
    cluster = H.Cluster(world.emu, n)
    out, errs = [None] * n, []

    def main(rank):
        H._tls.world, H._tls.m = H.World(cluster, rank), ModelM(cluster, world)
        w = H._tls.world
        try:
            with _lock:
                torch.manual_seed(0)
                model = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.Linear(64, 10)).bfloat16()
            shadow = [torch.nn.Parameter(p.detach().float().clone()) for p in model.parameters()]
            oracle = ps.SGD([(f"p{i}", q) for i, q in enumerate(shadow)], shadow, engine="host", use_mpi=False, **hyper)
            for h in oracle._hooks:
                h.remove()
            groups = oracle._group_of()
            opt = ps.SGD(model.named_parameters(), model.parameters(), mode="ps", engine="device", **hyper)
            layer = convert_first_linear(model, opt, relu=True, pull=pull, gate=True)
            assert isinstance(layer, BcastLinear) and model[0] is layer
            eng = opt._engine
            for s in range(steps):
                g = torch.Generator().manual_seed(10 * rank + s)
                x, y = torch.randn(8, 32, generator=g).bfloat16(), torch.randint(0, 10, (8,), generator=g)
                opt.zero_grad(set_to_none=True)
                torch.nn.functional.cross_entropy(model(x).float(), y).backward()
                mine = [p.grad.detach().float().clone() for p in model.parameters()]
                opt.step()
                allg = w.all_gather_object(mine)
                with torch.no_grad():
                    for i, q in enumerate(shadow):
                        oracle.optim_step(q, sum(allg[r][i] for r in range(n)), **oracle._hyper(groups[id(q)]))
            eng.ensure_params()
            eng.check()
            w.barrier()
            got = [(opt.state[p]["master_param"] if eng.master is not None else p).detach().float().clone()
                   for p in model.parameters()]
            res = dict(got=got, pub=[p.detach().clone() for p in model.parameters()], shadow=[q.detach().clone() for q in shadow],
                       log=list(H._tls.m.log), direct=set(eng.direct_names), server=eng.is_server)
            opt.close()
            oracle.close()
            out[rank] = res
        except BaseException as exc:       # noqa: BLE001
            errs.append(exc)
            cluster.fail(exc)

    ts = [threading.Thread(target=main, args=(r,), daemon=True) for r in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in ts), "a rank thread is stuck"
    if errs:
        real = [e for e in errs if "another rank" not in str(e) and not isinstance(e, threading.BrokenBarrierError)]
        raise (real or errs)[0]
    for r, res in enumerate(out):
        for a, b in zip(res["pub"], out[0]["pub"]):
            assert torch.equal(a, b)
        if res["server"]:
            for g, q in zip(res["got"], res["shadow"]):
                assert torch.allclose(g, q, rtol=2e-4, atol=2e-5), float((g - q).abs().max())
        assert "0.weight" in res["direct"]                                  # dW of the gated layer skipped the encode pass
        waits = [e for e in res["log"] if e[0] == "wait" and e[1] == H.M.SIG_PARAMS_READY]
        gates = [e[1] for e in res["log"] if e[0] == "gate"]
        if r > 0:
            assert len(waits) == 1 and gates == list(range(1, steps)), (waits, gates)


def test_tiny_bert_topk_adam_with_never_used_heads(world):
    """BASELINE config 4 in miniature: the package's BERT (tied decoder: one hook for two uses of the embedding matrix; the pooler
    and NSP head get NO gradient when only the MLM loss is trained → inactive parameters on every step), block-wise top-k wire,
    Adam with per-parameter step counts, bf16 parameters with fp32 masters, 2 ranks — against the grad-gather oracle."""
    n, steps = 2, 3
    hyper = dict(lr=1e-2, eps=1e-8, weight_decay=1e-2)
    cluster = H.Cluster(world.emu, n)
    out, errs = [None] * n, []

    def main(rank):
        H._tls.world, H._tls.m = H.World(cluster, rank), ModelM(cluster, world)
        w = H._tls.world
        try:
            with _lock:
                torch.manual_seed(0)
                model = models.bert_base(vocab_size=97, hidden_size=32, num_hidden_layers=2, num_attention_heads=4,
                                         intermediate_size=64, max_position_embeddings=16).bfloat16()
            names = [k for k, _ in model.named_parameters()]
            shadow = [torch.nn.Parameter(p.detach().float().clone()) for p in model.parameters()]
            oracle = ps.Adam([(f"p{i}", q) for i, q in enumerate(shadow)], shadow, engine="host", use_mpi=False, **hyper)
            for h in oracle._hooks:
                h.remove()
            groups = oracle._group_of()
            opt = ps.Adam(model.named_parameters(), model.parameters(), mode="ps", engine="device", code=ps.TopK(ratio=0.25), **hyper)
            eng = opt._engine
            before = {k: p.detach().clone() for k, p in model.named_parameters()}
            for s in range(steps):
                g = torch.Generator().manual_seed(7 * rank + s)
                ids = torch.randint(0, 97, (4, 12), generator=g)
                lab = torch.where(torch.rand(4, 12, generator=g) < 0.3, ids, torch.full_like(ids, -100))
                lab[0, 0] = ids[0, 0]
                opt.zero_grad(set_to_none=True)
                model(ids, mlm_labels=lab, nsp_labels=None).backward()
                mine = [None if p.grad is None else p.grad.detach().clone() for p in model.parameters()]
                opt.step()
                allg = w.all_gather_object(mine)
                with torch.no_grad():
                    for i, q in enumerate(shadow):
                        if allg[0][i] is None:
                            continue
                        total = torch.zeros_like(q)
                        for r in range(n):
                            code = ps.TopK(ratio=0.25)
                            total += code.decode(code.encode(allg[r][i], name=f"p{i}")).reshape(q.shape).float()
                        oracle.optim_step(q, total, **oracle._hyper(groups[id(q)]))
            eng.check()
            w.barrier()
            got = [(opt.state[p]["master_param"] if eng.master is not None else p).detach().float().clone()
                   for p in model.parameters()]
            sd = opt.state_dict()
            res = dict(names=names, got=got, shadow=[q.detach().clone() for q in shadow], server=eng.is_server,
                       pub={k: p.detach().clone() for k, p in model.named_parameters()}, before=before,
                       steps=[int(st.get("step", 0)) for st in sd["state"].values()] if eng.is_server else None)
            opt.close()
            oracle.close()
            out[rank] = res
        except BaseException as exc:       # noqa: BLE001
            errs.append(exc)
            cluster.fail(exc)

    ts = [threading.Thread(target=main, args=(r,), daemon=True) for r in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in ts), "a rank thread is stuck"
    if errs:
        real = [e for e in errs if "another rank" not in str(e) and not isinstance(e, threading.BrokenBarrierError)]
        raise (real or errs)[0]
    for res in out:
        unused = [k for k in res["names"] if k.startswith("nsp.") or "pooler" in k]
        assert len(unused) == 4
        for k in res["names"]:
            assert torch.equal(res["pub"][k], out[0]["pub"][k])                     # ranks identical
            assert torch.equal(res["pub"][k], res["before"][k]) == (k in unused), k   # never-used heads untouched, the rest moved
        if res["server"]:
            for k, g, q in zip(res["names"], res["got"], res["shadow"]):
                assert torch.allclose(g, q, rtol=2e-4, atol=2e-5), (k, float((g - q).abs().max()))
            assert sorted(set(res["steps"])) == [0, steps]                           # per-parameter step counts
