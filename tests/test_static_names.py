"""Cheap static check (no linters in this image): every name loaded inside the functions of the GPU-only host code is
bound somewhere visible.  Guards the paths that cannot execute on the CPU box (bench.py's GPU arm, runtime.py, worker.py)."""
import ast
import builtins
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = ["bench.py", "__graft_entry__.py", "flashmoe_b200/runtime.py", "flashmoe_b200/worker.py", "flashmoe_b200/_C.py",
         "flashmoe_b200/launcher.py", "flashmoe_b200/layer.py", "flashmoe_b200/ops.py", "flashmoe_b200/_lib.py", "flashmoe_b200/_build.py",
         "scripts/diag.py", "scripts/trace_gantt.py", "scripts/trace_multi.py", "tests/multi_gpu_worker.py"]


def _bound_names(node):
    names = set()
    for n in ast.walk(node):
        if isinstance(n, ast.Name) and isinstance(n.ctx, (ast.Store, ast.Del)):
            names.add(n.id)
        elif isinstance(n, (ast.FunctionDef, ast.AsyncFunctionDef, ast.ClassDef)):
            names.add(n.name)
        elif isinstance(n, ast.arg):
            names.add(n.arg)
        elif isinstance(n, (ast.Import, ast.ImportFrom)):
            for a in n.names:
                names.add((a.asname or a.name).split(".")[0])
        elif isinstance(n, ast.ExceptHandler) and n.name:
            names.add(n.name)
        elif isinstance(n, (ast.Global, ast.Nonlocal)):
            names.update(n.names)
    return names


def _check(tree):
    module_names = _bound_names(tree) | set(dir(builtins)) | {"__file__", "__name__", "__package__"}
    problems = []

    def visit(fn, outer):
        scope = outer | _bound_names(fn)
        for n in ast.walk(fn):
            if isinstance(n, ast.Name) and isinstance(n.ctx, ast.Load) and n.id not in scope:
                problems.append((fn.name, n.id, n.lineno))

    for node in ast.walk(tree):
        if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef)):
            visit(node, module_names)
    return problems


@pytest.mark.parametrize("rel", FILES)
def test_no_undefined_names(rel):
    tree = ast.parse(open(os.path.join(ROOT, rel)).read(), filename=rel)
    assert _check(tree) == []
