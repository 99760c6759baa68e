"""CPU: every FP8 cast and FP8 GEMM of the package is issued from the engine methods that own the FP8 linears.

tests/test_gpu_fp8_linears_elementwise.py checks each FP8 linear of a training step by spying on `_linear` and
`_linear_bwd_fp8` and counting the fp8 GEMM launches.  A call site anywhere else would run FP8 arithmetic those spies
cannot see; this test finds it by parsing the sources, without a GPU."""

import ast
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PACKAGE = os.path.join(ROOT, "dolomite_engine_b200")

FP8_ENTRY_POINTS = {"fp8_cast", "gemm_fp8", "gemm_fp8_wgrad_multi"}
# (module, class, method) allowed to issue them
OWNERS = {("engine.py", "DolomiteEngine", m) for m in ("_linear", "_fp8_weight", "_linear_bwd_fp8", "_flush_wgrads")}


def _sources():
    for d, _, files in os.walk(PACKAGE):
        for f in sorted(files):
            if f.endswith(".py"):
                yield os.path.relpath(os.path.join(d, f), PACKAGE)


def _uses(tree):
    """(name, line, enclosing (class, method) or None) of every reference to an FP8 entry point outside its definition:
    attribute access (K.gemm_fp8, kernels.gemm_fp8) and bare names (from .kernels import gemm_fp8) alike"""
    found = []

    def visit(node, owner):
        for child in ast.iter_child_nodes(node):
            o = owner
            if isinstance(node, ast.ClassDef) and isinstance(child, (ast.FunctionDef, ast.AsyncFunctionDef)):
                o = (node.name, child.name)
            elif isinstance(child, (ast.FunctionDef, ast.AsyncFunctionDef)) and owner is None:
                o = (None, child.name)
            if isinstance(child, ast.Attribute) and child.attr in FP8_ENTRY_POINTS:
                found.append((child.attr, child.lineno, o))
            elif isinstance(child, ast.Name) and child.id in FP8_ENTRY_POINTS:
                found.append((child.id, child.lineno, o))
            elif isinstance(child, ast.ImportFrom):
                found.extend((a.name, child.lineno, o) for a in child.names if a.name in FP8_ENTRY_POINTS)
            visit(child, o)

    visit(tree, None)
    return found


def test_fp8_entry_points_are_called_only_by_the_fp8_linear_methods():
    seen = set()
    outside = []
    for rel in _sources():
        with open(os.path.join(PACKAGE, rel)) as f:
            tree = ast.parse(f.read(), rel)
        for name, line, owner in _uses(tree):
            if owner is not None and (rel, *owner) in OWNERS:
                seen.add(name)
            else:
                outside.append(f"{rel}:{line} {name} in {owner}")
    assert not outside, outside
    # the scan finds the engine's own call sites (it is not looking at the wrong files or names)
    assert seen == FP8_ENTRY_POINTS


def test_scan_sees_nested_and_imported_call_sites():
    src = (
        "from .kernels import gemm_fp8\n"
        "class DolomiteEngine:\n"
        "    def _flush_wgrads(self):\n"
        "        def launch():\n"
        "            K.gemm_fp8_wgrad_multi([])\n"
        "    def other(self):\n"
        "        kernels.fp8_cast(x)\n"
        "def helper():\n"
        "    gemm_fp8(a)\n"
    )
    uses = _uses(ast.parse(src))
    assert uses == [("gemm_fp8", 1, None), ("gemm_fp8_wgrad_multi", 5, ("DolomiteEngine", "_flush_wgrads")),
                    ("fp8_cast", 7, ("DolomiteEngine", "other")), ("gemm_fp8", 9, (None, "helper"))]
