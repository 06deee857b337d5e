"""Every Python call into the native extension is bound — statically — against the signature pybind11 recorded in the BUILT
``.so``: a stale binary or a call site that drifted from ``bindings.cpp`` / ``gemm_bindings.cpp`` fails here, on the CPU, instead
of as a ``TypeError: incompatible function arguments`` on the GPU box (the extension imports without a GPU)."""
import ast
import inspect
import os
import re

import pytest

from tests.test_static_names import ROOT, _sources

RECEIVERS = {"m", "self.m", "ext.cuda()", "_ext.cuda()", "_C", "mod"}
PLAN_RECEIVERS = {"self.plan", "P", "plan"}
BLOCK_RECEIVERS = {"blk"}


def _signature(doc):
    """``inspect.Signature`` from the first line of a pybind11 docstring (``name(a: T, b: T = 0) -> R``)."""
    line = doc.strip().split("\n")[0]
    inner = line[line.index("(") + 1: line.rindex(") ->")]
    params, depth, cur = [], 0, ""
    for ch in inner:
        depth += ch in "[(" 
        depth -= ch in "])"
        if ch == "," and depth == 0:
            params.append(cur)
            cur = ""
        else:
            cur += ch
    if cur.strip():
        params.append(cur)
    out = []
    for p in params:
        name = p.split(":")[0].strip()
        if name == "self":
            continue
        has_default = re.search(r"=\s*[^=]+$", p.split(":", 1)[1]) is not None if ":" in p else False
        out.append(inspect.Parameter(name, inspect.Parameter.POSITIONAL_OR_KEYWORD,
                                     default=0 if has_default else inspect.Parameter.empty))
    return inspect.Signature(out)


@pytest.fixture(scope="module")
def native():
    from pytorch_ps_mpi_b200.ops import ext
    try:
        return ext.cuda()
    except Exception as exc:      # noqa: BLE001
        pytest.skip(f"extension not importable here: {exc}")


def _calls():
    for path in _sources():
        rel = os.path.relpath(path, ROOT)
        if rel.startswith("scratch/"):
            continue
        src = open(path).read()
        if ".cuda()" not in src or "ext" not in src:        # only files that obtain the extension module
            continue
        tree = ast.parse(src, path)
        for n in ast.walk(tree):
            if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute):
                yield rel, n, ast.unparse(n.func.value), n.func.attr


def test_every_native_call_site_binds(native):
    fns = {n: getattr(native, n) for n in dir(native) if not n.startswith("_") and callable(getattr(native, n))}
    plan = {n: getattr(native.UpdatePlan, n) for n in dir(native.UpdatePlan) if not n.startswith("_")}
    blk = {n: getattr(native.SymmBlock, n) for n in dir(native.SymmBlock) if not n.startswith("_")}
    checked, problems = 0, []
    for rel, call, recv, attr in _calls():
        table = fns if recv in RECEIVERS else plan if recv in PLAN_RECEIVERS else blk if recv in BLOCK_RECEIVERS else None
        if table is None:
            continue
        if attr not in table:
            if recv in ("m", "self.m", "ext.cuda()", "_ext.cuda()") and not attr.isupper():
                problems.append(f"{rel}:{call.lineno}: the extension has no function {attr!r}")
            continue
        obj = table[attr]
        if not callable(obj) or not getattr(obj, "__doc__", None) or "(" not in obj.__doc__:
            continue
        sig = _signature(obj.__doc__)
        names = list(sig.parameters)
        kw = {k.arg for k in call.keywords if k.arg is not None}
        unknown = kw - set(names)
        if unknown:
            problems.append(f"{rel}:{call.lineno}: {attr}() has no parameter(s) {sorted(unknown)}")
            continue
        if any(isinstance(a, ast.Starred) for a in call.args) or any(k.arg is None for k in call.keywords):
            checked += 1
            continue                       # *args / **kwargs: keyword names checked above, arity is dynamic
        try:
            sig.bind(*[0] * len(call.args), **{k: 0 for k in kw})
        except TypeError as exc:
            problems.append(f"{rel}:{call.lineno}: {attr}{sig}: {exc}")
        checked += 1
    assert not problems, "\n".join(problems)
    assert checked >= 30, checked          # the scan really saw the engine's call sites


def test_launch_mode_names_match_the_extension(native):
    """The engine's launch-mode constants mirror the enums of ``common.cuh`` that the extension exports."""
    from pytorch_ps_mpi_b200.parallel import device_engine as de
    names = [n for n in dir(de) if n.split("_")[0] in ("OPT", "BCAST", "REDUCE", "SIGNAL")]
    assert len(names) == 10
    assert {n: getattr(native, n) for n in names} == {n: getattr(de, n) for n in names}


def test_signature_parser():
    s = _signature("f(self: X, a: typing.SupportsInt | typing.SupportsIndex, b: collections.abc.Sequence[int] = [], "
                   "c: typing.SupportsFloat = 30.0) -> None\n")
    assert list(s.parameters) == ["a", "b", "c"]
    assert s.parameters["a"].default is inspect.Parameter.empty and s.parameters["c"].default == 0
    with pytest.raises(TypeError):
        s.bind()
    s.bind(1, c=2)
