"""CPU: the coverage table of ``tests/test_gpu_training_gradients.py`` stays complete.

Walks the package's syntax trees for classes with an ``autograd.Function`` base, however it is spelled (``Function``,
``autograd.Function``, ``torch.autograd.Function``, next to other bases), and fails when one has no row in
``BACKWARD_REACHED``, when a row names a class the package does not define, when a row names a variant the file does not
run, or when a Function no variant reaches has no reason in ``NOT_DIFFERENTIATED``.  A Function added later without a row fails
here, on a machine without a GPU."""
import ast
import os

from tests.test_gpu_training_gradients import _ALL, BACKWARD_REACHED, NOT_DIFFERENTIATED

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "swapping_autoencoder_pytorch_b200")


def _base_name(node):
    """the last component of a base-class expression: Function, autograd.Function, torch.autograd.Function -> "Function" """
    if isinstance(node, ast.Attribute):
        return node.attr
    if isinstance(node, ast.Name):
        return node.id
    return None


def _function_classes():
    found = {}
    for root, _, files in os.walk(PKG):
        for f in files:
            if f.endswith(".py"):
                path = os.path.join(root, f)
                with open(path) as fh:
                    tree = ast.parse(fh.read(), path)
                for node in ast.walk(tree):
                    if isinstance(node, ast.ClassDef) and any(_base_name(b) == "Function" for b in node.bases):
                        found[node.name] = os.path.relpath(path, PKG)
    return found


def test_every_function_has_a_row():
    found = _function_classes()
    assert len(found) >= 27, sorted(found)
    assert set(found) == set(BACKWARD_REACHED), ("no row:", sorted(set(found) - set(BACKWARD_REACHED)),
                                                 "row without a class:", sorted(set(BACKWARD_REACHED) - set(found)))


def test_parser_sees_every_spelling_of_the_base():
    src = ("class A(Function): pass\nclass B(autograd.Function): pass\nclass C(torch.autograd.Function): pass\n"
           "class D(Mixin, Function): pass\nclass E(Module): pass\n")
    names = {n.name for n in ast.walk(ast.parse(src))
             if isinstance(n, ast.ClassDef) and any(_base_name(b) == "Function" for b in n.bases)}
    assert names == {"A", "B", "C", "D"}


def test_rows_name_real_variants_and_unreached_ones_have_reasons():
    for name, variants in BACKWARD_REACHED.items():
        assert set(variants) <= set(_ALL), (name, variants)
    unreached = {name for name, variants in BACKWARD_REACHED.items() if not variants}
    assert unreached == set(NOT_DIFFERENTIATED), (sorted(unreached), sorted(NOT_DIFFERENTIATED))
    assert all(reason.strip() for reason in NOT_DIFFERENTIATED.values())
