"""The inventory of the workspace contract, on the host: every entry point of include/recnn_b200.h that takes a caller
workspace (void* workspace, int64_t workspace_bytes) and every *_record_floats query must appear in the COVERED table
of test_workspace_bounds_serving_gpu.py, naming a test that exists.  A new entry point that no bounds test runs fails
here, without a GPU."""
from __future__ import annotations

import ast
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "recnn_b200.h")
GPU_FILE = os.path.join(HERE, "test_workspace_bounds_serving_gpu.py")
DECL = re.compile(r"RECNN_API\s+[\w\s\*]*?\b(recnn_\w+)\s*\(([^;]*?)\)\s*;", re.S)
WORKSPACE = re.compile(r"void\s*\*\s*workspace\s*,\s*int64_t\s+workspace_bytes")


def declarations():
    """name -> parameter text of every RECNN_API declaration of the header"""
    with open(HEADER) as fh:
        text = re.sub(r"/\*.*?\*/", " ", fh.read(), flags=re.S)
    return {m.group(1): m.group(2) for m in DECL.finditer(text)}


def must_cover(decls):
    return {name for name, params in decls.items() if WORKSPACE.search(params) or name.endswith("_record_floats")}


def module_tree(path):
    with open(path) as fh:
        return ast.parse(fh.read(), path)


def covered_table(tree):
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "COVERED" for t in node.targets):
            return ast.literal_eval(node.value)
    raise AssertionError("no COVERED table in %s" % GPU_FILE)


def defined_tests(tree):
    return {n.name for n in tree.body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")}


def test_the_header_parses_into_the_expected_families():
    decls = declarations()
    need = must_cover(decls)
    # a parser that stopped matching would make the inventory vacuous
    assert len(decls) > 100, len(decls)
    for name in ("recnn_retrieve_topk_sets", "recnn_retrieve_rank_sets", "recnn_critic_topk", "recnn_critic_rank",
                 "recnn_discrete_shard_sample_topk_sets", "recnn_beta_shard_log_prob_stats",
                 "recnn_vocab_topk_record_floats", "recnn_discrete_value_dp_record_floats"):
        assert name in need, name
    assert "recnn_slate_distances" not in need and "recnn_ddpg_step" not in need


def test_every_workspace_and_record_entry_point_is_covered():
    decls = declarations()
    table = covered_table(module_tree(GPU_FILE))
    missing = sorted(must_cover(decls) - set(table))
    assert not missing, "entry points with a size contract that no bounds test runs: %s" % missing
    stale = sorted(set(table) - set(decls))
    assert not stale, "COVERED names entry points the header does not declare: %s" % stale


def test_every_covering_test_exists():
    trees = {}
    for name, where in covered_table(module_tree(GPU_FILE)).items():
        path, fn = where.split("::") if "::" in where else (os.path.basename(GPU_FILE), where)
        if path not in trees:
            trees[path] = defined_tests(module_tree(os.path.join(HERE, path)))
        assert fn in trees[path], "%s: %s has no test %s" % (name, path, fn)
