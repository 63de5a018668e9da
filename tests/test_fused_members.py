"""The solo solve's per-tile member lists (classes.cuh: list_member_index; fused.cuh: fused_select): the slot tiles write,
per class list, the registry positions of its members in tile order, and the selection picks the j-th member of a tile
with one load.  The cases sit at the index's edges: a class that owns every slot of a tile (j = 0 .. 1023), lists that
start, end or skip at tile boundaries, a last slot tile that is only partly filled, dead slots between live ones
(servants that are partly busy, below the batch's min_version or with max_tasks = 0), and more classes than one chunk of
lists (kListChunk) holds.  Every stream is replayed through the CUDA backend -- plain, packed and staged calls -- and
compared with the CPU checker; the YDSCHED_DEBUG solve lines show that it reached the speculative solve (variant 4) and
the solo solve that keeps its class table (variants 2 / 3).  Each case also runs next to a wide table whose list offsets
do not fit in shared memory, where the solo solve selects from the leader's scanned offsets."""
import numpy as np
import pytest

from yadcc_b200 import Servant
from yadcc_b200 import streams as S
from solve_lines import solves

pytestmark = pytest.mark.gpu


def _digests(k):
    return [f"{0x3e3b0000 + i:064x}" for i in range(k)]


def _servant(i: int, digests: list, version: int = 10, max_tasks: int = 24) -> Servant:
    return Servant(f"{S.servant_ip(i)}:8335", None, digests, version, 64, 0, 256 << 30, 200 << 30, max_tasks)


# name -> (servants as (digest index, version, max_tasks) per servant, number of digests, requests per batch, the
# digests the batches ask for, the share of its grants each batch frees before the next)
def _case(name):
    if name == "full-tile":
        # one class, 64 servants x 24 slots = 1536 slots: it owns every slot of tile 0 and half of tile 1, and a batch
        # asks for more than that (j runs through 0 .. 1023 in tile 0)
        return [(0, 10, 24)] * 64, 1, 2000, [0], 0.5
    if name == "boundaries":
        # one class with 32 slots per servant, one with 2 (its list ends in the first slot tile), one with 8: lists that
        # end early and skip the later tiles; 1024 + 64 + 128 slots, so the last tile is partly filled
        sv = [(0, 10, 32)] * 32 + [(1, 10, 2)] * 32 + [(2, 10, 8)] * 16
        return sv, 3, 1500, [0, 1, 2], 0.3
    if name == "dead-slots":
        # servants below the batches' min_version (8), servants with max_tasks = 0 and partly busy servants (only part
        # of each batch's grants is freed) between live ones
        sv = [(i % 4, 5 if i % 5 == 1 else 10, 0 if i % 7 == 3 else 16 + i % 9) for i in range(120)]
        return sv, 4, 1200, [0, 1, 2, 3], 0.4
    if name == "many-classes":
        # 80 classes, one component each: the kept table's slot tiles count their lists in two chunks of 64
        return [(i % 80, 10, 24) for i in range(160)], 80, 1000, list(range(80)), 0.5
    raise ValueError(name)


# 130 more digests on 520 servants of capacity 64, each digest asked for twice per batch: the class bound grows to 256
# and the static slot bound passes 33 800 slots (64 slot tiles), so the list offsets, 256 x 65 + 1 words, no longer fit
# in shared memory (16 384 words)
WIDE_DIGESTS, WIDE_SERVANTS, WIDE_ASKS = 130, 520, 2


def _stream(d, name, wide, seed=3):
    servants, n_digests, n_case, asked, free = _case(name)
    wide_asks = []
    if wide:
        servants = servants + [(n_digests + i % WIDE_DIGESTS, 10, 64) for i in range(WIDE_SERVANTS)]
        wide_asks = list(range(n_digests, n_digests + WIDE_DIGESTS)) * WIDE_ASKS
        n_digests += WIDE_DIGESTS
    n = n_case + len(wide_asks)
    dg = _digests(n_digests)
    ev = [("hb", 0.0, _servant(i, [dg[k]], v, mt), 100.0) for i, (k, v, mt) in enumerate(servants)]
    env = np.asarray([d.intern_env(x) for x in dg], dtype=np.uint32)
    outside = np.asarray([d.intern_ip(f"172.16.3.{i}") for i in range(100)], dtype=np.uint32)
    rng = np.random.default_rng(seed)
    now = 0.001
    for _ in range(7):  # one class set: the first solves keep the class table, the later ones speculate
        e = env[np.asarray(asked)[rng.integers(0, len(asked), n_case)]]
        if wide:
            e = rng.permutation(np.concatenate([e, env[wide_asks]]))
        ips = outside[rng.integers(0, len(outside), n)]
        ev.append(("wait", now, S._requests(d, e, ips, np.full(n, 8, np.uint32), expires_in_s=15.0,
                                            prefetch=rng.random(n) < 0.2)))
        ev.append(("state",))
        ev.append(("free_frac", int(rng.integers(1 << 30)), free))
        ev.append(("tick", now + 0.005))
        now += 0.01
    return S.Stream(f"members-{name}", ev), n


@pytest.mark.parametrize("selection", ["lite", "leader-scan"])
@pytest.mark.parametrize("mode", ["plain", "packed", "staged"])
@pytest.mark.parametrize("case", ["full-tile", "boundaries", "dead-slots", "many-classes"])
def test_member_lists_equal_oracle(make_dispatcher, monkeypatch, capfd, case, mode, selection):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    wide = selection == "leader-scan"
    traces = {}
    for kind in ("cuda", "port"):
        d = make_dispatcher(kind)
        stream, n = _stream(d, case, wide)
        cuda = kind == "cuda"
        traces[kind] = S.Replayer(d, pinned=cuda, packed=(mode == "packed" and cuda),
                                  staged=(mode == "staged" and cuda)).run(stream)
        d.close()
    assert S.traces_equal(traces["cuda"], traces["port"]), S.first_mismatch(traces["cuda"], traces["port"])
    lines = [x for x in solves(capfd.readouterr().err) if x["n"] == n]
    variants = [x["variant"] for x in lines]
    assert set(variants) & {2, 3}, variants  # the solo solve that keeps the class table ...
    if wide:
        assert 4 not in variants, variants  # (no speculation without the block-local tables)
        assert all(x["cls_bound"] * (x["slot_b"] // 1024 + 1) + 1 > 16384 for x in lines if x["variant"] in (2, 3)), lines
    else:
        assert any(x["variant"] == 4 and x["spec"] == 1 for x in lines), variants  # ... and the speculative one
