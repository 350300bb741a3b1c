"""CPU: a numpy model of the sharded grouped search protocol (DESIGN.md section 4.14) -- round 1 (each rank's own top G
groups with their best P rows), merge 1 (the best head per group id, the first G by (distance, global row)), round 2 (a
rank copies a chosen group it listed, scores one it holds but did not list, pads the rest) and merge 2 (each group's best
P rows over the ranks) -- must give exactly the whole-corpus grouped answer, for any world size, grouping, ties and
row filter.  Groups that never straddle a shard boundary must need no round-2 scoring."""
import numpy as np
import pytest

from wax_b200.sharded import shard_range


def grouped(rows, dist, gid, top_groups, per_group):
    """Grouped search over the given rows (all allowed, finite): [(group id, [(distance, global row), ...])], groups
    ranked by their best row in (distance, row), ties to the lower row; each group's best per_group rows."""
    order = np.lexsort((rows, dist))
    rows, dist, gid = rows[order], dist[order], gid[order]
    _, first = np.unique(gid, return_index=True)
    out = []
    for g in gid[np.sort(first)][:top_groups]:
        sel = gid == g
        out.append((int(g), list(zip(dist[sel][:per_group].tolist(), rows[sel][:per_group].tolist()))))
    return out


def protocol(dist, gid, allowed, world, top_groups, per_group):
    """The sharded answer and the number of (group, rank) pairs round 2 scored."""
    n = dist.size
    ok = allowed & np.isfinite(dist)
    shards = [shard_range(n, world, r) for r in range(world)]
    # round 1: every rank's own answer, with global rows
    local = []
    for lo, hi in shards:
        rows = np.arange(lo, hi)[ok[lo:hi]]
        local.append(grouped(rows, dist[rows], gid[rows], top_groups, per_group))
    # merge 1: the union of the heads, the best per group id, the first G by (distance, global row)
    best = {}
    for lst in local:
        for g, hits in lst:
            if g not in best or hits[0] < best[g]:
                best[g] = hits[0]
    chosen = sorted(best, key=lambda g: best[g])[:top_groups]
    if per_group == 1:
        return [(g, [best[g]]) for g in chosen], 0
    # round 2: copy, expand or pad; merge 2: each group's best per_group rows over the ranks
    expanded = 0
    answer = []
    for g in chosen:
        pooled = []
        for r, (lo, hi) in enumerate(shards):
            listed = dict(local[r])
            if g in listed:
                pooled += listed[g]
            elif np.any(gid[lo:hi] == g):
                expanded += 1
                rows = np.arange(lo, hi)[(gid[lo:hi] == g) & ok[lo:hi]]
                pooled += sorted(zip(dist[rows].tolist(), rows.tolist()))[:per_group]
        answer.append((g, sorted(pooled)[:per_group]))
    return answer, expanded


N = 600


def groupings(rng, world):
    edges = [shard_range(N, world, r)[0] for r in range(1, world)]
    straddle = np.zeros(N, np.int64)            # a group around every shard boundary, 5-row groups elsewhere
    for e in edges:
        straddle[max(e - 3, 0):e + 3] = -1 - e
    straddle = np.where(straddle < 0, straddle, np.arange(N) // 5 + 10_000)
    return {
        "contiguous": np.arange(N) // 8,
        "straddling": straddle,
        "hashed": (np.arange(N) * 2654435761 % 4093) % 97,
        "giant": np.zeros(N, np.int64),
        "unset": np.arange(N) + 5_000,            # every frame its own group (group id = frame id)
    }


def distances(rng, kind):
    if kind == "random":
        return rng.standard_normal(N).astype(np.float32)
    if kind == "tied":                             # a handful of values: ties within and across every shard
        return rng.integers(0, 6, N).astype(np.float32)
    return np.tile(rng.standard_normal(37).astype(np.float32), N // 37 + 1)[:N]   # period duplicates


@pytest.mark.parametrize("world", list(range(1, 17)))
def test_protocol_equals_the_whole_corpus_answer(world):
    rng = np.random.default_rng(world)
    for kind in ("random", "tied", "period"):
        dist = distances(rng, kind)
        dist[rng.choice(N, 5, replace=False)] = np.inf            # rows without a finite distance never take part
        for name, gid in groupings(rng, world).items():
            for mask in ("all", "random", "sparse"):
                allowed = {"all": np.ones(N, bool), "random": rng.random(N) < 0.6,
                           "sparse": rng.random(N) < 0.05}[mask]
                for top_groups in (1, 12, 256):
                    for per_group in (1, 3, 128):
                        rows = np.flatnonzero(allowed & np.isfinite(dist))
                        want = grouped(rows, dist[rows], gid[rows], top_groups, per_group)
                        got, _ = protocol(dist, gid, allowed, world, top_groups, per_group)
                        assert got == want, (world, kind, name, mask, top_groups, per_group)


@pytest.mark.parametrize("world", [2, 3, 5, 8, 16])
def test_groups_inside_one_shard_need_no_scoring(world):
    """A group held by one rank only is listed by that rank whenever it is chosen, so round 2 only copies; a group
    across a boundary may have to be scored on the rank that did not list it."""
    rng = np.random.default_rng(100 + world)
    dist = rng.standard_normal(N).astype(np.float32)
    allowed = np.ones(N, bool)
    lo_of = np.array([shard_range(N, world, r)[0] for r in range(world)])
    rank_of = np.searchsorted(lo_of, np.arange(N), side="right") - 1
    aligned = rank_of * 1000 + (np.arange(N) - lo_of[rank_of]) // 7        # consecutive groups cut at every boundary
    for top_groups in (1, 12, 256):
        for per_group in (3, 128):
            _, expanded = protocol(dist, aligned, allowed, world, top_groups, per_group)
            assert expanded == 0
    straddle = groupings(rng, world)["straddling"]
    edge = shard_range(N, world, 1)[0]
    dist[edge - 3:edge] -= 10.0            # the group across the first boundary ranks first by its rows below it ...
    _, expanded = protocol(dist, straddle, allowed, world, 1, 3)
    assert expanded == 1                   # ... so the rank above lists its own best group and scores this one
