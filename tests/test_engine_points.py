"""The lookahead engine configurations the fp64 replay tests run beyond bench.py's points (tools/engine_record.py ENGINE_POINTS)
follow what tools/pairnet_bench.py and tools/lookahead_cache_bench.py measure: every (shape, engine) those tools run has a
configuration, pairnet_bench.py's smallest and largest group at each shape are among them, lookahead_cache_bench.py's points appear
with its feature cache, and no configuration runs a shape neither tool runs.  Runs without a GPU: it reads the tools' tables and
the defaults of their arguments."""
import ast
import os
import re

from tools import lookahead_cache_bench as cache_bench
from tools import pairnet_bench
from tools.engine_record import ENGINE_POINTS, POINTS, point_config

TOOLS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")

# groups of pairnet_bench.py that need no configuration of their own, and why
STANDS_IN = {
    # (c2, batch 1, lookahead 1): maps of 8x8 and larger at batch 1 (trunk batch 3, decoder batch 1) are what bench.py's batch-1
    # points replay already; c1's smallest group is the smallest one that reaches maps (4x4) and batches no other configuration does
    ("c2", 1, 1): "pairnet_c1_b1_t1",
}


def _default(module, flag):
    with open(os.path.join(TOOLS, os.path.basename(module.__file__))) as f:
        m = re.search(r'add_argument\("%s",[^)]*?default=("[^"]*"|[-\w.]+)' % re.escape(flag), f.read())
    assert m, "%s has no default for %s" % (module.__name__, flag)
    return [int(v) for v in str(ast.literal_eval(m.group(1))).split(",")]


def _shape(cfg):
    return cfg["height"], cfg["width"], cfg["n_depth_levels"], cfg["n_measurement_frames"]


def _has(table, engine, shape, **want):
    """keys of the configurations of `table` (keys of ENGINE_POINTS) that run `engine` at `shape` with every field of `want` (a
    list: one of its values)"""
    cfgs = {k: point_config(k) for k in table}
    return [k for k, c in cfgs.items() if c["engine"] == engine and _shape(c) == shape and
            all(c[f] in v if isinstance(v, list) else c[f] == v for f, v in want.items())]


def required():
    """(what the tools measure, the fields a configuration must have) for every configuration the table needs"""
    out = []
    batches, lookaheads = _default(pairnet_bench, "--batches"), pairnet_bench.LOOKAHEADS
    for name, (H, W, D, M) in pairnet_bench.POINTS.items():
        shape = (H, W, D, M)
        out.append(("pairnet_bench.py %s" % name, ("pairnet", shape, {})))
        for B, T in ((min(batches), min(lookaheads)), (max(batches), max(lookaheads))):
            if (name, B, T) not in STANDS_IN:
                out.append(("pairnet_bench.py %s batch %d lookahead %d" % (name, B, T),
                            ("pairnet", shape, dict(batch=B, lookahead=T, feature_cache=0, terms=1))))
    cache_lookaheads = _default(cache_bench, "--lookaheads")
    for name, (H, W, D, M, pairnet) in cache_bench.POINTS.items():
        engine, shape = ("pairnet" if pairnet else "lookahead"), (H, W, D, M)
        out.append(("lookahead_cache_bench.py %s" % name, (engine, shape, {})))
        out.append(("lookahead_cache_bench.py %s with its feature cache" % name,
                    (engine, shape, dict(batch=1, feature_cache=[max(30, T * (M + 1)) for T in cache_lookaheads]))))
    return out


def unmet(table):
    """what the tools measure that no configuration of `table` runs"""
    return [what for what, (engine, shape, want) in required() if not _has(table, engine, shape, **want)]


def test_every_measured_engine_configuration_is_replayed():
    print()
    for what, (engine, shape, want) in required():
        print("%-62s %s" % (what, _has(ENGINE_POINTS, engine, shape, **want) or "NOT REPLAYED"))
    assert not unmet(ENGINE_POINTS), "configurations the tools measure that no replay runs: %s" % unmet(ENGINE_POINTS)
    assert not set(POINTS) & set(ENGINE_POINTS), "keys in both tables: %s" % sorted(set(POINTS) & set(ENGINE_POINTS))
    for stands_for, key in STANDS_IN.items():
        assert key in ENGINE_POINTS and point_config(key)["lookahead"] * point_config(key)["batch"] == 1, (stands_for, key)


def test_no_configuration_runs_a_shape_no_tool_runs():
    shapes = {s for s in pairnet_bench.POINTS.values()} | {s[:4] for s in cache_bench.POINTS.values()}
    stray = {k: _shape(point_config(k)) for k in ENGINE_POINTS if _shape(point_config(k)) not in shapes}
    assert not stray, "configurations at shapes neither tool runs: %s" % stray
    for k in ENGINE_POINTS:
        cfg = point_config(k)
        assert cfg["engine"] in ("pairnet", "lookahead"), (k, cfg["engine"])
        if cfg["feature_cache"]:
            assert cfg["feature_cache"] >= cfg["lookahead"] * (cfg["n_measurement_frames"] + 1), (k, cfg)


def test_removing_a_configuration_is_reported():
    expect = {"pairnet_c1_b1_t1": "pairnet_bench.py c1 batch 1 lookahead 1",
              "pairnet_c1_b8_t8": "pairnet_bench.py c1 batch 8 lookahead 8",
              "pairnet_c2_b8_t8": "pairnet_bench.py c2 batch 8 lookahead 8",
              "pairnet_c1_b1_t8_cache": "lookahead_cache_bench.py pairnet-c1 with its feature cache",
              "pairnet_c2_b1_t4_cache": "lookahead_cache_bench.py pairnet-c2 with its feature cache",
              "fusionnet_c2_t4_cache": "lookahead_cache_bench.py fusionnet-c2",
              "fusionnet_c3_t4_cache": "lookahead_cache_bench.py fusionnet-c3"}
    for k, what in expect.items():
        missing = unmet({p: v for p, v in ENGINE_POINTS.items() if p != k})
        assert what in missing, "removing %s is not reported (%s)" % (k, missing)
