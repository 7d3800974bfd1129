"""Every operating point bench.py reports is replayed against the fp64 references: its key is in tools/engine_record.py's POINTS (the
engine configurations the replay tests of tests/test_tc_reference.py, tests/test_engine_coverage.py and tests/test_sweep_reference.py
run over), or in NON_KERNEL_POINTS with the test that covers it.  Also, every plane-sweep batch of bench.py's roofline
is a case of tests/test_sweep_reference.py.  Runs without a GPU: it reads bench.py's source."""
import ast
import os
import re

from tools.engine_record import NON_KERNEL_POINTS, POINTS

BENCH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py")


def _source():
    with open(BENCH) as f:
        return f.read()


def _default(src, flag):
    m = re.search(r'add_argument\("%s",[^)]*?default=("[^"]*"|[-\w.]+)' % re.escape(flag), src)
    assert m, "bench.py has no default for %s" % flag
    return ast.literal_eval(m.group(1))


def _expansions(src):
    """the keys bench.py formats at run time, as its default arguments spell them"""
    B = _default(src, "--clips")
    return {
        "batched_%d": ["batched_%d" % int(v) for v in str(_default(src, "--extra-clips")).split(",") if int(v) > B],
        "pipelined_%d_stages_no_lookahead": ["pipelined_%d_stages_no_lookahead" % _default(src, "--stages")],
        "operands_%s": ["operands_fp16_pairs_3_terms" if _default(src, "--tc-terms") == 1 else "operands_fp16_1_term"],
    }


def reported_points(src):
    """the headline ("value") and every key of bench.py's operating_points a default run reports"""
    assert re.search(r'"value": fps\b', src), "bench.py no longer reports its headline as \"value\""
    exp = _expansions(src)
    keys = ["value"]
    for k in re.findall(r'extras\[\s*"([^"]+)"', src):
        if "%" in k:
            assert k in exp, "bench.py reports a formatted key this test cannot expand: %s" % k
            keys += exp[k]
        else:
            keys.append(k)
    return list(dict.fromkeys(keys))


def unlisted(points, table=None):
    table = POINTS if table is None else table
    return [k for k in points if k not in table and k not in NON_KERNEL_POINTS]


def test_every_bench_point_is_replayed():
    points = reported_points(_source())
    print()
    for k in points:
        print("%-40s %s" % (k, POINTS.get(k) or "no kernel: " + NON_KERNEL_POINTS.get(k, "NOT REPLAYED")))
    assert not unlisted(points), "bench.py reports points no replay test runs: %s" % unlisted(points)
    assert not set(POINTS) & set(NON_KERNEL_POINTS)
    stale = sorted((set(POINTS) | set(NON_KERNEL_POINTS)) - set(points))
    assert not stale, "points bench.py does not report: %s" % stale
    assert {"batched_8", "batched_32", "config_c3_320x256_96planes_4frames", "operands_fp16_pairs_3_terms"} <= set(points)


def test_removing_a_point_is_reported():
    points = reported_points(_source())
    for k in ("batched_32", "config_c3_320x256_96planes_4frames", "feature_cache", "value"):
        assert unlisted(points, {p: v for p, v in POINTS.items() if p != k}) == [k]


def test_roofline_batches_are_sweep_cases():
    from tests.test_sweep_reference import CASES
    src = _source()
    m = re.search(r"for nb in \(B, ([\d, ]+)\):", src)
    assert m, "bench.py's roofline batches moved"
    for nb in [_default(src, "--clips")] + [int(v) for v in m.group(1).split(",") if v.strip()]:
        assert CASES.get("roofline_%d" % nb) == (nb, 128, 128, 64, 2), "bench.py times the sweep at nb=%d: no such case" % nb
