"""Every CUDA graph of the package is captured by engine.capture_graphs, so the warm-up and restore rule lives in one place: no other
module constructs a torch.cuda.CUDAGraph or enters torch.cuda.graph."""
import ast
import os

from conftest import ROOT

PKG = os.path.join(ROOT, "diff-pruning_b200")
CAPTURE = {"torch.cuda.CUDAGraph", "torch.cuda.graph"}


def _dotted(node):
    parts = []
    while isinstance(node, ast.Attribute):
        parts.append(node.attr)
        node = node.value
    if isinstance(node, ast.Name):
        parts.append(node.id)
        return ".".join(reversed(parts))
    return None


def _capture_calls():
    """{module path relative to the package: [(line, dotted name)]} of every call to torch.cuda.CUDAGraph / torch.cuda.graph."""
    found = {}
    for d, _, files in os.walk(PKG):
        for f in sorted(files):
            if not f.endswith(".py"):
                continue
            path = os.path.join(d, f)
            with open(path) as fh:
                tree = ast.parse(fh.read(), path)
            for node in ast.walk(tree):
                if isinstance(node, ast.Call) and _dotted(node.func) in CAPTURE:
                    found.setdefault(os.path.relpath(path, PKG), []).append((node.lineno, _dotted(node.func)))
    return found


def test_graphs_are_captured_in_engine_only():
    found = _capture_calls()
    assert set(found) == {"engine.py"}, {k: v for k, v in found.items() if k != "engine.py"}
    assert sorted(name for _, name in found["engine.py"]) == sorted(CAPTURE), found["engine.py"]
