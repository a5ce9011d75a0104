"""No test file imports another: a gate, a checker or a pinned list that more than one file needs lives in a module of
its own (engine_harness.py, launch_check.py, tile_check.py, the *_cases.py tables), not in whichever test file defined
it first."""
import ast
import glob
import os

TESTS = os.path.dirname(os.path.abspath(__file__))


def _imported(tree):
    """the dotted names of the modules a parsed file imports, whatever the import form"""
    for node in ast.walk(tree):
        if isinstance(node, ast.Import):
            yield from (a.name for a in node.names)
        elif isinstance(node, ast.ImportFrom) and node.level == 0 and node.module:
            yield node.module
            yield from ('%s.%s' % (node.module, a.name) for a in node.names)
        elif isinstance(node, ast.ImportFrom):                 # from . import test_x / from .test_x import y
            yield from ('tests.' + n for n in ([node.module] if node.module else [a.name for a in node.names]))


def test_no_test_file_imports_another():
    bad = []
    for path in sorted(glob.glob(os.path.join(TESTS, 'test_*.py'))):
        with open(path) as f:
            tree = ast.parse(f.read(), path)
        bad += ['%s imports %s' % (os.path.basename(path), m) for m in _imported(tree)
                if m.startswith('tests.test_')]
    assert not bad, bad
