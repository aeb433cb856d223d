"""The product never downloads: no module of unflow_b200 imports urllib or names a URL in its code
(the reference's dataset classes fetch missing datasets; these adapters only read local files)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATTERN = re.compile(r"urllib|urlretrieve|https?://")


def _code_lines(path):
    """Lines of ``path`` with comments stripped (citations in comments are not code)."""
    for n, line in enumerate(open(path, encoding='utf-8'), 1):
        code = line.split('//', 1)[0] if path.endswith(('.cu', '.cuh', '.h', '.cpp')) else line.split('#', 1)[0]
        yield n, code


def test_product_code_has_no_network_access():
    hits = []
    for base, _, files in os.walk(os.path.join(ROOT, "unflow_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                path = os.path.join(base, f)
                hits += ["%s:%d" % (os.path.relpath(path, ROOT), n) for n, code in _code_lines(path)
                         if PATTERN.search(code)]
    assert not hits, hits
