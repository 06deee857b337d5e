"""AdamW (``ps.AdamW``, decoupled weight decay) on both engines.

* the host engine against ``torch.optim.AdamW(foreach=False)``, bit for bit;
* optimizer rule A1 of ``DESIGN.md`` (a numpy replay) against torch: the moments bit for bit, the parameter equal wherever
  torch's vectorised CPU ``sqrt`` is correctly rounded;
* ``psb_update_kernel<…, OPT_ADAMW>`` through the real bindings against the replay, bit for bit (CPU emulator of the same
  source by default, the GPU with ``-m gpu``);
* the device engine on the emulator (real bindings) against a single-process oracle, and two engine ranks on one GPU."""
import contextlib
import copy

import numpy as np
import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200 import runtime
from pytorch_ps_mpi_b200.codings import KIND_DENSE, TILE, WIRE_F32
from pytorch_ps_mpi_b200.launch import spawn
from pytorch_ps_mpi_b200.parallel import device_engine as de
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout
from tests import _cuda_emu
from tests.test_multirank_engine_emulation import _attach, _data, _loss, _model, emu, run_ranks  # noqa: F401  (emu: fixture)

F32 = np.float32
DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
GDT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
OPT_ADAMW = 2
BPT = TILE * 4


# ---------------------------------------------------------------------------------------------------------------------
# the rule (DESIGN.md, optimizer rule A1) in numpy
# ---------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 fused multiply-add rounded once: the product is exact in float64, the float64 sum is rounded to odd, then to
    fp32 (53 >= 24 + 2 bits, so the two roundings give the correctly rounded result)."""
    a, b, c = (np.asarray(x, F32).astype(np.float64) for x in (a, b, c))
    p = a * b
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        fix = np.isfinite(s) & (e != 0) & ((s.view(np.uint64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def scalars(lr, wd, betas, eps, t):
    """The fp32 scalars of step ``t``: each formed in double and rounded once."""
    b1, b2 = betas
    return dict(d=F32(1 - lr * wd), a=F32(1 - b1), a2=F32(1 - b2), b2=F32(b2), eps=F32(eps), s=F32(lr / (1 - b1 ** t)),
                c2=F32((1 - b2 ** t) ** 0.5))


def rule(w, m, v, vm, g, h, amsgrad, sqrt=np.sqrt):
    """One step of rule A1 on fp32 arrays; returns (w, m, v, vm).  ``sqrt`` is the correctly rounded root by default."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if h["d"] != 1:
            w = (w * h["d"]).astype(F32)
        if h["a"] < 0.5:
            m = fma32(h["a"], (g - m).astype(F32), m)
        else:
            m = fma32(F32(h["a"] - F32(1)), (g - m).astype(F32), g)
        v = fma32((h["a2"] * g).astype(F32), g, (v * h["b2"]).astype(F32))
        vh = v
        if amsgrad:
            vm = np.maximum(vm, v)                                 # NaN propagates, as torch.maximum
            vh = vm
        den = ((sqrt(vh).astype(F32) / h["c2"]).astype(F32) + h["eps"]).astype(F32)
        w = (w + ((-h["s"] * m).astype(F32) / den).astype(F32)).astype(F32)
    return w, m, v, vm


def bits(x):
    return np.asarray(x, F32).view(np.uint32)


def same_bits(a, b):
    """Bit for bit, except that any NaN equals any NaN (its sign and payload are the processor's: the GPU returns the
    canonical NaN)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(bits(a[~nan]), bits(b[~nan]))


# ---------------------------------------------------------------------------------------------------------------------
# 1. host engine == torch.optim.AdamW(foreach=False)
# ---------------------------------------------------------------------------------------------------------------------
def _net():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.LayerNorm(32), torch.nn.Tanh(), torch.nn.Linear(32, 4))


def _groups(model):
    """BERT-style groups: matrices decay, biases and LayerNorm parameters do not."""
    dec = [p for p in model.parameters() if p.dim() == 2]
    nod = [p for p in model.parameters() if p.dim() != 2]
    return [{"params": dec}, {"params": nod, "weight_decay": 0.0}]


@pytest.mark.parametrize("amsgrad", [False, True])
def test_host_engine_bit_identical_to_torch(amsgrad):
    runtime.init()
    a, b = _net(), _net()
    mine = ps.AdamW(a.named_parameters(), _groups(a), lr=1e-2, weight_decay=0.05, amsgrad=amsgrad, engine="host")
    ref = torch.optim.AdamW(_groups(b), lr=1e-2, weight_decay=0.05, amsgrad=amsgrad, foreach=False)
    assert mine._engine is None and mine.optim == "adamw" and mine.defaults["weight_decay"] == 0.05
    for step in range(7):
        x = torch.randn(8, 16, generator=torch.Generator().manual_seed(step))
        for model, opt in ((a, mine), (b, ref)):
            opt.zero_grad(set_to_none=True)
            out = model[:2](x).sum() if step == 2 else model(x).square().sum()     # step 2: the head gets no gradient
            out.backward()
            opt.step()
        if step == 3:                                                               # an lr change mid-run
            for g in mine.param_groups + ref.param_groups:
                g["lr"] = 3e-3
        for p, q in zip(a.parameters(), b.parameters()):
            assert torch.equal(p, q), step
    for p, q in zip(a.parameters(), b.parameters()):
        for k, v in ref.state[q].items():
            assert torch.equal(mine.state[p][k], v), k
    mine.close()


def test_defaults_and_maximize():
    runtime.init()
    model = _net()
    opt = ps.AdamW(model.named_parameters(), model.parameters(), engine="host")
    assert opt.defaults["weight_decay"] == 1e-2 and opt.defaults["betas"] == (0.9, 0.999)
    opt.close()
    with pytest.raises(ValueError, match="maximize"):
        ps.AdamW(model.named_parameters(), model.parameters(), maximize=True, engine="host")


# ---------------------------------------------------------------------------------------------------------------------
# 2. the rule against torch on the CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("amsgrad", [False, True])
@pytest.mark.parametrize("hyper", [(1e-3, 1e-2, (0.9, 0.999), 1e-8), (3e-2, 0.1, (0.4, 0.99), 1e-6)])
def test_rule_against_torch(amsgrad, hyper):
    """``m`` and ``v`` bit-identical every step.  ``w`` also, once torch's own (vectorised, not always correctly rounded)
    ``sqrt`` replaces the correctly rounded one; with the correctly rounded root, ``w`` differs only in elements where torch's
    root is off, by one ulp of the root."""
    lr, wd, betas, eps = hyper
    rng = np.random.default_rng(5)
    n = 1 << 16
    w0 = rng.standard_normal(n).astype(F32)
    p = torch.nn.Parameter(torch.from_numpy(w0.copy()))
    ref = torch.optim.AdamW([p], lr=lr, weight_decay=wd, betas=betas, eps=eps, amsgrad=amsgrad, foreach=False)
    w, m, v, vm = w0.copy(), np.zeros(n, F32), np.zeros(n, F32), np.zeros(n, F32)
    torch_sqrt = lambda x: torch.from_numpy(np.ascontiguousarray(x)).sqrt().numpy()     # noqa: E731
    for t in range(1, 6):
        g = (10.0 ** rng.uniform(-6, 2, n) * rng.choice([-1, 1], n)).astype(F32)
        p.grad = torch.from_numpy(g)
        ref.step()
        h = scalars(lr, wd, betas, eps, t)
        w_t, m, v, vm = rule(w, m, v, vm, g, h, amsgrad, sqrt=torch_sqrt)
        st = ref.state[p]
        assert same_bits(m, st["exp_avg"].numpy()) and same_bits(v, st["exp_avg_sq"].numpy()), t
        assert same_bits(w_t, p.detach().numpy()), t
        # the kernel's rule, from the same start: differs only where torch's root is not correctly rounded
        vh = vm if amsgrad else v
        off = bits(np.sqrt(vh)) != bits(torch_sqrt(vh))
        h_den = lambda r: ((r.astype(F32) / h["c2"]).astype(F32) + h["eps"]).astype(F32)      # noqa: E731
        w_dec = (w * h["d"]).astype(F32) if h["d"] != 1 else w
        w_c = (w_dec + ((-h["s"] * m).astype(F32) / h_den(np.sqrt(vh))).astype(F32)).astype(F32)
        diff = bits(w_c) != bits(w_t)
        assert not (diff & ~off).any(), t
        assert diff.sum() <= off.sum() and off.sum() < n // 50, (int(diff.sum()), int(off.sum()))
        w = w_t


# ---------------------------------------------------------------------------------------------------------------------
# 3. psb_update_kernel<KIND_DENSE, WIRE_F32, OPT_ADAMW> against the rule, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
class Ranks:
    """N virtual ranks over the real bindings: fp32 gradient wires (the sum is exact to replay), two parameter groups
    (decayed, and ``weight_decay=0``), optimizer state over tiles ``[lo, ntiles)`` kept compactly (``state_shift = lo``)."""

    NUMELS = (3 * TILE + 99, 700, 2 * TILE, 5)

    def __init__(self, be, dtype, nranks, lo=0):
        if be == "gpu":
            from pytorch_ps_mpi_b200.ops import ext
            self.m, self.dev = ext.cuda(), torch.device("cuda", 0)
        else:
            self.m, self.dev = _cuda_emu.build_extension(), torch.device("cpu")
            if self.m is None:
                pytest.skip("no g++")
        self.be, self.n, self.dtype, self.lo = be, nranks, dtype, lo
        self.params = [torch.nn.Parameter(torch.zeros(k, dtype=dtype)) for k in self.NUMELS]
        groups = [{"params": self.params[:2]}, {"params": self.params[2:]}]
        self.L = L = FlatLayout(groups, {id(p): f"p{i}" for i, p in enumerate(self.params)})
        self.slots = [L.by_id[id(p)] for p in self.params]
        nt, npad = L.ntiles, L.numel_padded
        self.real = np.zeros(npad, bool)
        for s in self.slots:
            self.real[s.offset: s.offset + s.numel] = True
        z = lambda k, dt: torch.zeros(k, dtype=dt, device=self.dev)      # noqa: E731
        self.tiles = L.tile_table_fast().to(self.dev)
        self.group_of = np.repeat(L.tile_table_fast()[:, 2].numpy(), TILE)
        self.param_of = np.repeat(L.tile_table_fast()[:, 0].numpy(), TILE)
        self.wires = [z(nt * BPT, torch.uint8) for _ in range(nranks)]
        self.scales = [z(L.nparams, torch.float32) for _ in range(nranks)]
        self.arenas = [z(npad, dtype) for _ in range(nranks)]
        self.signals = [z(512, torch.int64) for _ in range(nranks)]
        ns = (nt - lo) * TILE
        self.master = z(ns, torch.float32) if dtype != torch.float32 else None
        self.buf0, self.buf1, self.buf2 = z(ns, torch.float32), z(ns, torch.float32), z(ns, torch.float32)
        self.counters = z(8, torch.int32)
        P = self.m.UpdatePlan()
        P.kind, P.wire, P.opt = KIND_DENSE, WIRE_F32, self.m.OPT_ADAMW
        P.grid = min(nt - lo, 3 if be == "emu" else self.m.update_max_grid(KIND_DENSE, WIRE_F32, P.opt))
        for r in range(nranks):
            P.set_rank_ptrs(r, self.wires[r].data_ptr(), self.scales[r].data_ptr(), self.arenas[r].data_ptr(),
                            self.signals[r].data_ptr())
        P.configure(nranks, 0, nt, BPT, TILE, DT[dtype], 1 if nranks > 1 else 0, 0, 0, 0, self.arenas[0].data_ptr(),
                    self.master.data_ptr() if self.master is not None else 0, self.buf0.data_ptr(), self.buf1.data_ptr(),
                    self.buf2.data_ptr(), self.tiles.data_ptr(), self.signals[0].data_ptr(), self.counters.data_ptr(),
                    self.counters.data_ptr() + 4)
        self.P = P

    def set_start(self, full):
        t = torch.from_numpy(full)
        for a in self.arenas:
            a.copy_(t.to(self.dtype))
        if self.master is not None:
            self.master.copy_(t.to(self.dtype).float()[self.lo * TILE:])
        return t.to(self.dtype).float().numpy()

    def encode(self, r, full):
        grads = [torch.from_numpy(np.ascontiguousarray(full[s.offset: s.offset + s.numel])).to(self.dev) for s in self.slots]
        S = self.slots
        self.m.encode(KIND_DENSE, WIRE_F32, grads, [s.first_tile for s in S], [s.ntiles for s in S], [s.index for s in S],
                      self.tiles.data_ptr(), self.wires[r].data_ptr(), 0, 0, 0, BPT, 0, 1.0)

    def update(self, hypers, average, param_hyper=None, active=None):
        """One launch over tiles [lo, ntiles); ``param_hyper``: per-parameter {s, c2}; ``active``: per-parameter 0 / 1."""
        ph = act = 0
        if param_hyper is not None:
            self._ph = torch.from_numpy(param_hyper).to(self.dev)
            ph = self._ph.data_ptr()
        if active is not None:
            self._act = torch.tensor(active, dtype=torch.uint8, device=self.dev)
            act = self._act.data_ptr()
        self.P.launch(1, hypers, (1 << self.n) - 1, (1.0 / self.n) if average else 1.0, 0, 1, timeout_s=5.0, active_ptr=act,
                      tile_begin=self.lo, tile_end=self.L.ntiles, param_hyper=ph, **({"state_shift": self.lo} if self.lo else {}))
        if self.be == "gpu":
            torch.cuda.synchronize()

    def state(self, t):
        return t.cpu().float().numpy()


BACKENDS = ["emu", pytest.param("gpu", marks=pytest.mark.gpu)]
HYP = [dict(lr=2e-2, wd=0.1, betas=(0.9, 0.999), eps=1e-8), dict(lr=1e-2, wd=0.0, betas=(0.6, 0.95), eps=1e-6)]


def _group_tuple(hp, t, amsgrad):
    b1, b2 = hp["betas"]
    return [hp["lr"], 1 - hp["lr"] * hp["wd"], 1 - b1, 1 - b2, (1 - b2 ** t) ** 0.5, b2, hp["eps"], hp["lr"] / (1 - b1 ** t),
            0.0, float(amsgrad), 0.0]


def _kernel_case(be, pname, world, amsgrad=False, average=False, late=False, lo=0, nan=False, steps=3):
    dtype = GDT[pname]
    V = Ranks(be, dtype, world, lo=lo)
    rng = np.random.default_rng(world * 31 + len(pname) + 7 * amsgrad + 3 * average + 5 * late + lo)
    npad, e_lo = V.L.numel_padded, lo * TILE
    w = V.set_start(np.where(V.real, rng.standard_normal(npad), 0).astype(F32))
    pub0 = [V.state(a).copy() for a in V.arenas]
    m, v, vm = (np.zeros(npad, F32) for _ in range(3))
    gid, pid = V.group_of, V.param_of
    psteps = np.zeros(len(V.slots), int)
    for t in range(1, steps + 1):
        skip = late and t == 1                                    # parameter 0 gets no gradient in step 1: it starts late
        tot = np.zeros(npad, F32)
        for r in range(world):
            g = np.where(V.real, rng.standard_normal(npad) * 10.0 ** rng.uniform(-4, 1, npad), 0).astype(F32)
            if nan and r == world - 1 and t == 2:
                g[V.slots[0].offset + TILE + 5] = np.nan if r % 2 else np.inf
                g[V.slots[2].offset + 17] = -np.inf
            V.encode(r, g)
            tot = (tot + g).astype(F32)                            # rank order, fp32
        if average:
            tot = (tot * F32(1.0 / world)).astype(F32)
        active = [not (skip and i == 0) for i in range(len(V.slots))]
        psteps += np.array(active, int)
        hypers = [_group_tuple(HYP[k], t, amsgrad) for k in range(2)]
        ph = None
        if late:
            ph = np.zeros((len(V.slots), 2), F32)
            for i, s in enumerate(V.slots):                      # (indexed like the tile table: by slot index)
                hp = HYP[s.group]
                t_i = max(int(psteps[i]), 1)                           # (an inactive parameter's entry is never read)
                ph[s.index] = (hp["lr"] / (1 - hp["betas"][0] ** t_i), (1 - hp["betas"][1] ** t_i) ** 0.5)
        act = [1] * len(V.slots)
        for i, s in enumerate(V.slots):
            act[s.index] = int(active[i])
        V.update(hypers, average, ph, active=act if skip else None)   # the engine's active mask
        # the replay, per group (and per parameter's own step count)
        nw, nm, nv, nvm = np.copy(w), np.copy(m), np.copy(v), np.copy(vm)
        for i, s in enumerate(V.slots):
            if not active[i]:
                continue
            sl = slice(s.first_tile * TILE, (s.first_tile + s.ntiles) * TILE)
            hp = HYP[s.group]
            h = scalars(hp["lr"], hp["wd"], hp["betas"], hp["eps"], int(psteps[i]) if late else t)
            nw[sl], nm[sl], nv[sl], nvm[sl] = rule(w[sl], m[sl], v[sl], vm[sl], tot[sl], h, amsgrad)
        w, m, v, vm = nw, nm, nv, nvm
        got_w = V.state(V.master) if V.master is not None else V.state(V.arenas[0])[e_lo:]
        tag = (be, pname, world, amsgrad, average, late, lo, t)
        assert same_bits(got_w, w[e_lo:]), tag + (np.flatnonzero(bits(got_w) != bits(w[e_lo:]))[:5].tolist(),)
        assert same_bits(V.state(V.buf0), m[e_lo:]) and same_bits(V.state(V.buf1), v[e_lo:]), tag
        if amsgrad:
            assert same_bits(V.state(V.buf2), vm[e_lo:]), tag
        else:
            assert (V.state(V.buf2) == 0).all(), tag
        assert (got_w[~V.real[e_lo:]] == 0).all(), tag                       # padding stays 0
        for r in range(world):
            pub = V.state(V.arenas[r])
            want = torch.from_numpy(w).to(dtype).float().numpy()
            if lo:
                assert same_bits(pub[:e_lo], pub0[r][:e_lo]), tag                # outside the window: untouched
            assert same_bits(pub[e_lo:], want[e_lo:]), tag
        if nan and t >= 2:
            for i in (0, 2):
                sl = slice(V.slots[i].offset, V.slots[i].offset + V.slots[i].numel)
                assert np.isnan(w[sl]).any() and np.isnan(got_w[sl.start - e_lo: sl.stop - e_lo]).any(), "NaN / Inf → NaN"
    return V


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("world", [1, 2, 5, 16])
@pytest.mark.parametrize("pname", ["fp32", "bf16", "fp16"])
def test_kernel_bits(be, world, pname):
    _kernel_case(be, pname, world, amsgrad=world % 2 == 0, average=world == 5)


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("case", ["amsgrad+average", "late", "nan", "compact", "compact+late"])
def test_kernel_cases(be, case):
    kw = {"amsgrad+average": dict(amsgrad=True, average=True), "late": dict(late=True, amsgrad=True), "nan": dict(nan=True),
          "compact": dict(lo=2, amsgrad=True), "compact+late": dict(lo=3, late=True)}[case]
    _kernel_case(be, "bf16" if "compact" in case else "fp32", 3, **kw)


def test_binding_checks_the_adamw_tuple():
    m = _cuda_emu.build_extension()
    if m is None:
        pytest.skip("no g++")
    assert m.OPT_ADAMW == OPT_ADAMW == de._OPTIMS["adamw"].code
    V = Ranks("emu", torch.float32, 1)
    bad = _group_tuple(HYP[0], 1, False)
    for c2 in (0.0, float("nan"), float("inf"), -1.0):
        bad[4] = c2
        with pytest.raises(RuntimeError, match="c2"):
            V.P.launch(1, [bad, bad], 1, 1.0, 0, 1, timeout_s=5.0)
    with pytest.raises(RuntimeError, match="11 entries"):
        V.P.launch(1, [bad[:10]], 1, 1.0, 0, 1, timeout_s=5.0)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the device engine on the emulator, through the real bindings
# ---------------------------------------------------------------------------------------------------------------------
HYPER = dict(lr=1e-2, weight_decay=0.05, amsgrad=True)


def _adamw_groups(model):
    return [{"params": [p for p in model.parameters() if p.dim() == 2]},
            {"params": [p for p in model.parameters() if p.dim() != 2], "weight_decay": 0.0}]


def _oracle(n, steps, skip_until=0, average=False):
    """One process: every rank's gradient summed in rank order, then ``ps.AdamW``'s host step (torch's sequence)."""
    model = _model()
    opt = ps.AdamW(model.named_parameters(), _adamw_groups(model), engine="host", **HYPER)
    for h in opt._hooks:
        h.remove()
    groups = opt._group_of()
    for s in range(steps):
        tot = None
        for r in range(n):
            model.zero_grad(set_to_none=True)
            _loss(model, *_data(r, s), skip_head=s < skip_until).backward()
            gs = [None if p.grad is None else p.grad.clone() for p in model.parameters()]
            tot = gs if tot is None else [a if b is None else a + b for a, b in zip(tot, gs)]
        with torch.no_grad():
            for p, g in zip(model.parameters(), tot):
                if g is not None:
                    opt.optim_step(p, g / n if average else g, **opt._hyper(groups[id(p)]))
    opt.close()
    return [p.detach().clone() for p in model.parameters()]


def _engine_run(emu, n, mode, steps=4, coding=None, micro=1, skip_until=0, average=False, body=None):
    def rank_main(rank, w):
        model = _model()
        opt = ps.AdamW(model.named_parameters(), _adamw_groups(model), engine="host", mode=mode, average=average,
                       code=coding() if coding else None, **({"quota": n - 1} if mode == "async" else {}), **HYPER)
        _attach(opt, reduce="p2p")
        eng = opt._engine
        assert eng.optim.code == OPT_ADAMW and (not eng.is_server or eng.plan.opt == OPT_ADAMW)
        if body is not None:
            return body(rank, w, model, opt)
        if mode == "async" and rank == 0:
            opt.serve()
        else:
            for s in range(steps):
                opt.zero_grad(set_to_none=True)
                for k in range(micro):                                 # the last micro-batch outside no_sync()
                    with opt.no_sync() if k < micro - 1 else contextlib.nullcontext():
                        _loss(model, *_data(rank * micro + k, s), skip_head=s < skip_until).backward()
                opt.step()
        eng.check()
        w.barrier()
        out = [p.detach().clone() for p in model.parameters()]
        opt.close()
        return out

    return run_ranks(emu, n, rank_main)


def _close(a, b, tol=2e-5):
    for x, y in zip(a, b):
        assert torch.allclose(x, y, rtol=tol, atol=tol * 0.1), float((x - y).abs().max())


def _equal(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("n,mode,average,skip_until", [(2, "ps", False, 0), (3, "ps", True, 2), (3, "allgather", False, 2)])
def test_engine_sync_modes_match_oracle(emu, n, mode, average, skip_until):
    res = _engine_run(emu, n, mode, skip_until=skip_until, average=average)
    _close(res[0], _oracle(n, 4, skip_until=skip_until, average=average))
    for r in res:
        _equal(r, res[0])                                              # ranks bit-identical
    if mode == "ps":
        _equal(_engine_run(emu, n, "sharded", skip_until=skip_until, average=average)[0], res[0])   # sharded == ps, bits


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_engine_async_applies_the_worker_gradients(emu):
    """Async with one worker and quota 1: the server applies each of the worker's gradients once, in order, as the host step
    does (the worker may compute them on stale parameters: they are recorded)."""
    def body(rank, w, model, opt):
        grads = []
        if rank == 0:
            opt.serve()
        else:
            for s in range(3):
                opt.zero_grad(set_to_none=True)
                _loss(model, *_data(1, s), skip_head=False).backward()
                grads.append([p.grad.clone() for p in model.parameters()])
                opt.step()
        opt.close()                                            # the workers' close() ends the server's serve()
        return [p.detach().clone() for p in model.parameters()], grads

    res = _engine_run(emu, 2, "async", body=body)
    model = _model()
    opt = ps.AdamW(model.named_parameters(), _adamw_groups(model), engine="host", **HYPER)
    groups = opt._group_of()
    for gs in res[1][1]:
        with torch.no_grad():
            for p, g in zip(model.parameters(), gs):
                opt.optim_step(p, g, **opt._hyper(groups[id(p)]))
    opt.close()
    _close(res[0][0], [p.detach() for p in model.parameters()])


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("coding", ["qsgd", "sign"])
def test_engine_coded_wire_sharded_equals_ps(emu, coding):
    code = {"qsgd": lambda: ps.QSGD(levels=7, blockwise=True), "sign": lambda: ps.Sign()}[coding]
    a = _engine_run(emu, 3, "ps", coding=code)
    b = _engine_run(emu, 3, "sharded", coding=code)
    _equal(a[0], b[0])
    for r in b:
        _equal(r, b[0])


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_engine_no_sync_last_micro_batch_outside(emu):
    """Two micro-batches, the last one outside ``no_sync()``: the same bits as both inside and ``step()`` after the block."""
    got = _engine_run(emu, 2, "ps", steps=3, micro=2)

    def all_inside(rank, w, model, opt):
        for s in range(3):
            opt.zero_grad(set_to_none=True)
            with opt.no_sync():
                for k in range(2):
                    _loss(model, *_data(rank * 2 + k, s), skip_head=False).backward()
            opt.step()
        opt._engine.check()
        w.barrier()
        out = [p.detach().clone() for p in model.parameters()]
        opt.close()
        return out

    want = _engine_run(emu, 2, "ps", body=all_inside)
    _equal(got[0], want[0])
    _equal(got[1], want[1])


def _train_steps(rank, model, opt, steps, first=0):
    for s in range(first, first + steps):
        opt.zero_grad(set_to_none=True)
        _loss(model, *_data(rank, s), skip_head=False).backward()
        opt.step()


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("first,second", [("ps", "ps"), ("ps", "sharded"), ("sharded", "ps")])
def test_engine_checkpoint_resume(emu, first, second):
    """Two steps, ``state_dict()`` (collective in ``sharded``), a fresh optimizer in the other mode loads it, two more steps:
    the same bits as four straight steps."""
    straight = _engine_run(emu, 2, "ps", steps=4)

    def body(rank, w, model, opt):
        _train_steps(rank, model, opt, 2)
        sd = copy.deepcopy(opt.state_dict())                  # collective in mode='sharded': every rank calls it
        sd = w.broadcast_object(sd, src=0)                    # written once (rank 0), loaded everywhere
        assert set(sd["state"][0]) >= {"step", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"}
        msd = {k: v.clone() for k, v in model.state_dict().items()}
        opt.close()
        model2 = _model()
        model2.load_state_dict(msd)
        opt2 = ps.AdamW(model2.named_parameters(), _adamw_groups(model2), engine="host", mode=second, **HYPER)
        _attach(opt2, reduce="p2p")
        opt2.load_state_dict(sd)
        _train_steps(rank, model2, opt2, 2, first=2)
        opt2._engine.check()
        w.barrier()
        out = [p.detach().clone() for p in model2.parameters()]
        opt2.close()
        return out

    got = _engine_run(emu, 2, first, body=body)
    _equal(got[0], straight[0])
    _equal(got[1], straight[1])


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_engine_checkpoint_to_torch_and_back(emu):
    """A one-rank engine checkpoint continues in ``torch.optim.AdamW``; torch's checkpoint (tensor steps) continues in the
    engine; both stay within fp32 rounding of an all-torch run."""
    def body(rank, w, model, opt):
        _train_steps(rank, model, opt, 2)
        sd = copy.deepcopy(opt.state_dict())
        msd = {k: v.clone() for k, v in model.state_dict().items()}
        opt.close()
        tmodel = _model()
        tmodel.load_state_dict(msd)
        ref = torch.optim.AdamW(_adamw_groups(tmodel), foreach=False, **HYPER)
        ref.load_state_dict(sd)
        _train_steps(rank, tmodel, ref, 2, first=2)
        sd2 = copy.deepcopy(ref.state_dict())
        assert torch.is_tensor(sd2["state"][0]["step"])
        model2 = _model()
        model2.load_state_dict(tmodel.state_dict())
        opt2 = ps.AdamW(model2.named_parameters(), _adamw_groups(model2), engine="host", **HYPER)
        _attach(opt2, reduce="p2p")
        opt2.load_state_dict(sd2)
        _train_steps(rank, model2, opt2, 2, first=4)
        opt2._engine.check()
        out = [p.detach().clone() for p in model2.parameters()]
        opt2.close()
        return out

    got = _engine_run(emu, 1, "ps", body=body)[0]
    model = _model()
    ref = torch.optim.AdamW(_adamw_groups(model), foreach=False, **HYPER)
    _train_steps(0, model, ref, 6)
    _close(got, [p.detach() for p in model.parameters()])


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_adam_and_adamw_ranks_refused(emu):
    def rank_main(rank, w):
        model = _model()
        cls = ps.Adam if rank == 0 else ps.AdamW
        opt = cls(model.named_parameters(), model.parameters(), engine="host", mode="ps", lr=1e-2)
        with pytest.raises(ValueError, match="optimizer"):
            _attach(opt)
        opt.close()
        return True

    assert run_ranks(emu, 2, rank_main) == [True, True]


# ---------------------------------------------------------------------------------------------------------------------
# 5. the GPU: two engine ranks on one H100, a tiny BERT with the no-decay group
# ---------------------------------------------------------------------------------------------------------------------
def _bert_groups(model):
    nod = [p for n, p in model.named_parameters() if n.endswith("bias") or "LayerNorm" in n or "_ln" in n or ".ln" in n
           or "norm" in n.lower()]
    ids = {id(p) for p in nod}
    return [{"params": [p for p in model.parameters() if id(p) not in ids]}, {"params": nod, "weight_decay": 0.0}]


def _tiny_bert():
    from pytorch_ps_mpi_b200.models import bert
    torch.manual_seed(0)
    return bert.bert_base(vocab_size=512, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128,
                          max_position_embeddings=64)


def _bert_batch(rank, s, dev):
    g = torch.Generator().manual_seed(100 * rank + s)
    ids = torch.randint(0, 512, (4, 32), generator=g)
    lab = torch.where(torch.rand(4, 32, generator=g) < 0.3, ids, torch.full_like(ids, -100))
    return ids.to(dev), lab.to(dev), torch.randint(0, 2, (4,), generator=g).to(dev)


def gpu_bert_ranks(rank, size, mode, reduce="p2p"):
    w = runtime.init()
    dev = w.device
    model = _tiny_bert().to(dev)
    groups = _bert_groups(model)
    assert groups[1]["params"]
    opt = ps.AdamW(model.named_parameters(), groups, mode=mode, engine="device", reduce=reduce, lr=1e-3, weight_decay=0.01)
    eng = opt._engine
    assert eng is not None and eng.m.OPT_ADAMW == eng.optim.code == OPT_ADAMW
    assert eng.plan is None or eng.plan.opt == OPT_ADAMW                   # (in mode='ps' only rank 0 has an update plan)
    for s in range(4):
        opt.zero_grad(set_to_none=True)
        ids, lab, nsp = _bert_batch(rank, s, dev)
        model(ids, mlm_labels=lab, nsp_labels=nsp).backward()
        opt.step()
    opt._engine.ensure_params()
    opt._engine.check()
    torch.cuda.synchronize()
    got = torch.cat([p.detach().reshape(-1) for p in model.parameters()]).cpu()
    opt.close()
    every = w.all_gather_object(got)
    assert all(torch.equal(x, every[0]) for x in every), "ranks diverged"
    if rank == 0:
        # the host-engine oracle: the rank-ordered sum of every rank's gradient, then ps.AdamW's host step
        ref = _tiny_bert().to(dev)
        ro = ps.AdamW(ref.named_parameters(), _bert_groups(ref), engine="host", lr=1e-3, weight_decay=0.01, use_mpi=False)
        for h in ro._hooks:
            h.remove()
        gmap = ro._group_of()
        for s in range(4):
            tot = None
            for r in range(size):
                ref.zero_grad(set_to_none=True)
                ids, lab, nsp = _bert_batch(r, s, dev)
                ref(ids, mlm_labels=lab, nsp_labels=nsp).backward()
                gs = [p.grad.clone() for p in ref.parameters()]
                tot = gs if tot is None else [a + b for a, b in zip(tot, gs)]
            with torch.no_grad():
                for p, g in zip(ref.parameters(), tot):
                    ro.optim_step(p, g, **ro._hyper(gmap[id(p)]))
        want = torch.cat([p.detach().reshape(-1) for p in ref.parameters()]).cpu()
        ro.close()
        assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), float((got - want).abs().max())
        print("adamw bert ok", mode, size, flush=True)


ONE_GPU = {"PSB200_PG_BACKEND": "gloo", "CUDA_VISIBLE_DEVICES": "0", "PSB200_DEVICE_TIMEOUT": "20"}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["ps", "sharded"])
def test_gpu_tiny_bert_two_ranks_one_gpu(mode):
    spawn(gpu_bert_ranks, 2, (mode,), env=dict(ONE_GPU, PSB200_CHUNK_BYTES="65536"), timeout=300)


@pytest.mark.gpu
def test_gpu_multi_gpu_nvls():
    """Two or more GPUs: ``ps`` and ``sharded`` with the machine's default reduction (NVLS where the switch has it)."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    for mode in ("ps", "sharded"):
        spawn(gpu_bert_ranks, min(n, 8), (mode, "auto"), env={"PSB200_DEVICE_TIMEOUT": "20"}, timeout=300)
