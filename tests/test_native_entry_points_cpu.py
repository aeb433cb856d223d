"""Every entry point of libunflow.so is classified for the float64 launch checks (tests/native_entry_points.py)."""
import ast
import os

import native_entry_points as EP
from unflow_b200 import _native

HERE = os.path.dirname(os.path.abspath(__file__))


def test_every_entry_point_is_in_exactly_one_group():
    groups = {"step": set(EP.STEP_CHECKED), "tc": set(EP.TC_DELEGATED), "host": set(EP.HOST_ONLY),
              "standalone": set(EP.STANDALONE)}
    for name in _native.SIGNATURES:
        where = [g for g, names in groups.items() if name in names]
        assert len(where) == 1, "%s is in %s: put it in exactly one group of tests/native_entry_points.py" % (
            name, where or "no group")
    extra = set().union(*groups.values()) - set(_native.SIGNATURES)
    assert not extra, "not entry points of the library: %s" % sorted(extra)


def test_step_checkers_and_pinned_sets_match_the_table():
    src = open(os.path.join(HERE, "test_gpu_step_launches.py")).read()
    tree = ast.parse(src)
    checkers = next(n for n in tree.body if isinstance(n, ast.Assign) and n.targets[0].id == "CHECKERS")
    keys = {k.value for k in checkers.value.keys}
    assert keys == set(EP.STEP_CHECKED)
    for pinned in (EP.PLAIN_STEP_CALLS, EP.AUGMENT_STEP_CALLS):
        assert pinned <= set(EP.STEP_CHECKED) | set(EP.TC_DELEGATED) | set(EP.HOST_ONLY)


def _assigned_dict(tree, name):
    return next(n.value for n in tree.body if isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Name)
                and n.targets[0].id == name)


def test_variant_checkers_and_pinned_sets_match_the_table():
    tree = ast.parse(open(os.path.join(HERE, "test_gpu_variant_step_launches.py")).read())
    checkers = _assigned_dict(tree, "VARIANT_CHECKERS")
    spread = [v.id for k, v in zip(checkers.keys, checkers.values) if k is None]
    assert spread == ["CHECKERS"], "VARIANT_CHECKERS must extend the step's CHECKERS"
    assert {k.value for k in checkers.keys if k is not None} == set(EP.VARIANT_CHECKED)
    assert not set(EP.VARIANT_CHECKED) & set(EP.STEP_CHECKED)
    assert set(EP.VARIANT_CHECKED) <= set(EP.STANDALONE)
    configs = {k.value for k in _assigned_dict(tree, "CONFIGS").keys}
    assert configs == set(EP.VARIANT_STEP_CALLS) == {"C-chairs", "C-kitti1152", "S-synthia", "cs-cityscapes",
                                                     "CSS-bench", "CSS-ft-train_all"}
    checked = set(EP.STEP_CHECKED) | set(EP.VARIANT_CHECKED) | set(EP.TC_DELEGATED) | set(EP.HOST_ONLY)
    for cid, pinned in EP.VARIANT_STEP_CALLS.items():
        assert pinned <= checked, "%s calls entry points without a checker: %s" % (cid, sorted(pinned - checked))


def test_standalone_entry_points_name_existing_tests():
    for name, ref in EP.STANDALONE.items():
        fname, test = ref.split("::")
        tree = ast.parse(open(os.path.join(HERE, fname)).read())
        funcs = {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}
        assert test in funcs, "%s: %s does not exist" % (name, ref)
        body = open(os.path.join(HERE, fname)).read()
        assert name[len("unflow_"):] in body or name in body or fname == "test_gpu_supervised.py" \
            or fname == "test_gpu_conv3x.py", "%s is not exercised in %s" % (name, fname)
