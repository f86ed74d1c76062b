"""vlm/dense.py is the only Python code in the package that calls the dense C-ABI entry points (GEMMs, LayerNorms, attention,
x2 split, casts): every engine goes through its wrappers instead of marshalling those ctypes calls itself."""
import ast
import os

from vlfm_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PACKAGE = os.path.join(ROOT, "vlfm_b200")
DENSE = os.path.join(PACKAGE, "vlm", "dense.py")
ENTRY_POINTS = {
    "vlfm_gemm_f16", "vlfm_gemm_f16_resid_ln", "vlfm_gemm_f16x2", "vlfm_gemm_f16x2_resid_ln", "vlfm_layernorm", "vlfm_layernorm_x2",
    "vlfm_attention_f16", "vlfm_attention_f32", "vlfm_split_x2", "vlfm_cast_f32_f16", "vlfm_cast_addpos_f16",
}


def entry_point_uses(path):
    """(line, name) of every `x.<entry point>` attribute and `getattr(x, "<entry point>")` in a Python file."""
    tree = ast.parse(open(path).read(), path)
    uses = []
    for node in ast.walk(tree):
        if isinstance(node, ast.Attribute) and node.attr in ENTRY_POINTS:
            uses.append((node.lineno, node.attr))
        elif (isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "getattr" and len(node.args) >= 2
              and isinstance(node.args[1], ast.Constant) and node.args[1].value in ENTRY_POINTS):
            uses.append((node.lineno, node.args[1].value))
    return uses


def test_entry_points_are_declared():
    assert ENTRY_POINTS <= set(_lib.declared_symbols())


def test_dense_wraps_every_entry_point():
    assert {name for _, name in entry_point_uses(DENSE)} == ENTRY_POINTS


def test_only_dense_calls_the_entry_points():
    offenders = []
    for d, _, files in os.walk(PACKAGE):
        for f in files:
            path = os.path.join(d, f)
            if f.endswith(".py") and path != DENSE:
                offenders += [f"{os.path.relpath(path, ROOT)}:{line}: {name}" for line, name in entry_point_uses(path)]
    assert not offenders, "call these through vlfm_b200/vlm/dense.py:\n" + "\n".join(offenders)
