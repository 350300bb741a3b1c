"""CPU: sharded.plan_rebalance (the rule the multi-device handle's wax_vs_rebalance ports to C++) against a brute-force
model over seeded count vectors, and the parts of wax_vs_rebalance that need no device: the NULL engine, the declaration
in both copies of the header and the C++ mirror's rebalance(), compiled and linked."""
import ctypes as C
import itertools
import subprocess
from pathlib import Path

import numpy as np
import pytest

from wax_b200 import _lib as L
from wax_b200 import build, sharded

ROOT = Path(__file__).resolve().parents[1]


def _count_vectors():
    rng = np.random.default_rng(20261018)
    for r in range(1, 17):
        yield [0] * r
        yield [7] * r
        yield list(range(r))
        for _ in range(12):
            hi = int(rng.choice([2, 5, 40, 1000]))
            yield rng.integers(0, hi, r).tolist()
        c = [0] * r                                  # everything on one shard
        c[int(rng.integers(0, r))] = int(rng.integers(1, 500))
        yield c


def _min_moved(counts):
    """The fewest rows any targets of T // R rows each, T % R of them one more, can move (brute force)."""
    total, r = sum(counts), len(counts)
    base, extra = divmod(total, r)
    best = None
    for plus in itertools.combinations(range(r), extra):
        t = [base + (i in plus) for i in range(r)]
        moved = sum(max(0, c - x) for c, x in zip(counts, t))
        best = moved if best is None else min(best, moved)
    return best


@pytest.mark.parametrize("counts", list(_count_vectors()))
def test_plan_against_a_brute_force_model(counts):
    targets, moves = sharded.plan_rebalance(counts)
    targets = [int(t) for t in targets]
    r, total = len(counts), sum(counts)
    assert sum(targets) == total and max(targets) - min(targets) <= 1
    # the extra rows sit on the shards that held the most, ties to lower shards
    base = total // r
    plus = [i for i in range(r) if targets[i] == base + 1]
    assert plus == sorted(sorted(range(r), key=lambda i: -counts[i])[:total % r])
    moved = sum(n for _, _, n in moves)
    assert moved == _min_moved(counts)
    assert all(n > 0 for _, _, n in moves)
    # donors give, receivers take, each in shard order, and the result is the targets
    assert moves == sorted(moves, key=lambda m: (m[0], m[1]))
    assert not {d for d, _, _ in moves} & {x for _, x, _ in moves}
    # replay on shards of keys: a donor loses only its tail, dealt out in key order to the receivers in shard order
    nxt = 0
    shards = []
    for c in counts:
        shards.append(list(range(nxt, nxt + c)))
        nxt += c
    rng = np.random.default_rng(sum(counts) + r)
    keys = rng.permutation(nxt)                      # keys interleave across shards; each shard's stay increasing
    shards = [sorted(keys[k].tolist() for k in s) for s in shards]
    tails = {d: shards[d][targets[d]:] for d in {d for d, _, _ in moves}}
    for d in tails:
        assert len(tails[d]) == counts[d] - targets[d]
    dealt = {d: [] for d in tails}
    for d, x, n in moves:
        run = shards[d][targets[d]:][len(dealt[d]):len(dealt[d]) + n]
        dealt[d] += run
        shards[x] = sorted(shards[x] + run)
    for d in tails:
        assert dealt[d] == tails[d]
        shards[d] = shards[d][:targets[d]]
    assert [len(s) for s in shards] == targets
    assert sorted(k for s in shards for k in s) == list(range(nxt))


@pytest.mark.parametrize("counts", [[0], [5], [3, 3], [4, 3, 4], [10, 9, 10, 10], [0, 1, 1, 0], [6] * 16])
def test_a_balanced_handle_moves_nothing(counts):
    targets, moves = sharded.plan_rebalance(counts)
    assert moves == [] and targets.tolist() == counts


def test_null_engine_without_a_device():
    moved = C.c_uint64(99)
    assert L.lib().wax_vs_rebalance(None, C.byref(moved)) == L.ERR_NULL
    assert L.last_error() == "engine is NULL" and moved.value == 0
    assert L.lib().wax_vs_rebalance(None, None) == L.ERR_NULL


def test_swift_header_copy_is_identical_and_declares_rebalance():
    a = (ROOT / "include" / "wax_vs_cuda.h").read_bytes()
    b = (ROOT / "swift" / "Sources" / "WaxVectorSearchCUDAC" / "include" / "wax_vs_cuda.h").read_bytes()
    assert a == b and b"int32_t wax_vs_rebalance(wax_vs_engine *engine, uint64_t *out_moved);" in a


def test_cxx_mirror_rebalance_links(tmp_path):
    lib = build.build()
    src = tmp_path / "probe.cpp"
    src.write_text(f'''#include <cstdio>
#include "{ROOT / "wax_b200" / "host" / "cuda_vector_engine.hpp"}"
int main() {{
    uint64_t (wax::CUDAVectorEngine::*fn)() = &wax::CUDAVectorEngine::rebalance;
    try {{
        wax::CUDAVectorEngine bad(wax::VectorMetric::cosine, 64, std::vector<int32_t>{{0, -1}});
        std::printf("%llu\\n", static_cast<unsigned long long>((bad.*fn)()));
        return 1;
    }} catch (const wax::WaxError &e) {{
        std::printf("%s\\n", e.what());
    }}
    return 0;
}}
''')
    exe = tmp_path / "probe"
    subprocess.run(["g++", "-std=c++17", "-Wall", str(src), f"-L{lib.parent}", "-lwaxvs_cuda", f"-Wl,-rpath,{lib.parent}",
                    "-o", str(exe)], check=True, capture_output=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "device ordinal -1 is negative" in out.stdout, (out.returncode, out.stdout, out.stderr)
