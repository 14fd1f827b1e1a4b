"""Randomised join pipelines: join type, number of keys, join qual, grouping side, aggregates and the planner's group
estimate (which decides between the on-chip variants and the HBM group table) drawn at random over relations with
duplicate and NULL keys; GPU vs oracle (the oracle's join is pinned by the nested loop of test_oracle_join.py)."""
import numpy as np
import pytest

from _util import assert_aggrows_match
from greengage_b200 import capi
from oracle import pyoracle as po
from test_gpu_join import gpu_joinagg
from test_oracle_join import ALL_JOINTYPES, join_nodes, small_relations

pytestmark = pytest.mark.gpu
BOTH = (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL)


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def random_join_case(seed):
    rng = np.random.default_rng(500 + seed)
    rel = small_relations(seed=int(rng.integers(0, 1000)), nouter=int(rng.integers(200, 3000)), ninner=int(rng.integers(1, 800)))
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = rel
    jointype = ALL_JOINTYPES[int(rng.integers(0, len(ALL_JOINTYPES)))]
    nkeys = int(rng.integers(1, 3))
    with_qual = bool(rng.random() < 0.4)
    p, outer, inner, hj = join_nodes(odesc, idesc, jointype, nkeys, with_qual)
    aggs = [(capi.AGG_COUNT_STAR, -1)]
    cands = [(capi.AGG_SUM_FLOAT8, p.var(3, capi.FLOAT8OID, 0)), (capi.AGG_MIN_FLOAT8, p.var(3, capi.FLOAT8OID, 0)), (capi.AGG_COUNT_ANY, p.var(1, capi.INT4OID, 0)),
             (capi.AGG_AVG_FLOAT8, p.var(3, capi.FLOAT8OID, 0))]
    keys = [[], [p.var(2, capi.BPCHAROID, 0)], [p.var(1, capi.INT4OID, 0)]]
    if jointype in BOTH:
        cands += [(capi.AGG_SUM_INT4, p.var(3, capi.INT4OID, 1)), (capi.AGG_MAX_INT4, p.var(3, capi.INT4OID, 1)), (capi.AGG_COUNT_ANY, p.var(2, capi.BPCHAROID, 1))]
        keys += [[p.var(2, capi.BPCHAROID, 1)], [p.var(1, capi.INT4OID, 1), p.var(2, capi.BPCHAROID, 0)]]
    for i in rng.permutation(len(cands))[:int(rng.integers(1, 4))]:
        aggs.append(cands[int(i)])
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, keys[int(rng.integers(0, len(keys)))], aggs, num_groups=int(rng.choice([0, 10, 500])))
    return outer, inner, hj, agg, p, opages, ipages, (jointype, nkeys, with_qual)


@pytest.mark.parametrize("seed", list(range(20)))
def test_random_join(eng, seed):
    outer, inner, hj, agg, p, opages, ipages, what = random_join_case(seed)
    want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, p.pool, opages, ipages, cap=20_000, exact=True)
    got, nj, _ = gpu_joinagg(eng, outer, inner, hj, agg, p.pool, opages, ipages, twice=(seed % 3 == 0))
    assert nj == nj_want, what
    assert_aggrows_match(got, want, agg, exact=want_x)
