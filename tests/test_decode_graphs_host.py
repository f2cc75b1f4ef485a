"""CUDA-graph steps of the paged decoder on the CPU: which steps are replayed and in which bucket, the step descriptor that the
plan kernel and the neighbour search read (against a pure-Python statement of where each new row goes), page rollback, and the
switch that turns the graphs off."""
import types

import numpy as np
import pytest
import torch

from se3_transformer_pytorch_b200 import ops, switches
from se3_transformer_pytorch_b200.model import DECODE_GRAPH_ROWS, PageTables, PagedCausalDecoder, decode_graph_bucket


# ---- eligibility and buckets ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,bucket', [(1, 1), (2, 2), (3, 4), (5, 8), (16, 16), (17, 32), (33, 64), (64, 64)])
def test_bucket_is_rows_rounded_up_to_a_power_of_two(M, bucket):
    seqlens = [1] * M if M <= 8 else [M - 3, 1, 2]
    assert decode_graph_bucket(100, [5] * len(seqlens), seqlens, [4] * len(seqlens)) == (bucket, 4)


@pytest.mark.parametrize('case', ['no_max_nodes', 'prompt', 'rows', 'mixed_k'])
def test_ineligible_steps_run_eagerly(case):
    n_prev, seqlens, ks, max_nodes = [5, 9], [1, 2], [4, 4], 100
    if case == 'no_max_nodes':
        max_nodes = None
    elif case == 'prompt':
        n_prev = [5, 0]                             # a cloud in its first call carries its prompt
    elif case == 'rows':
        seqlens = [DECODE_GRAPH_ROWS, 1]
    else:
        ks = [4, 3]
    assert decode_graph_bucket(max_nodes, n_prev, seqlens, ks) is None
    assert decode_graph_bucket(100, [5, 9], [DECODE_GRAPH_ROWS - 1, 1], [4, 4]) == (DECODE_GRAPH_ROWS, 4)


# ---- the descriptor ---------------------------------------------------------------------------------------------------------
def host_plan(desc, num_clouds, rows, P, scratch_row):
    """What se3_decode_plan_fwd writes, restated from se3b200.h: int64 [4, rows] of positions, pool rows, pair rows, clouds."""
    words = desc.numpy()
    nd = 5 * num_clouds + 1
    head = words[:2 * nd].view(np.int64)
    cu, n_prev = head[:num_clouds + 1], head[num_clouds + 1:2 * num_clouds + 1]
    pair_off, table_off = head[3 * num_clouds + 1:4 * num_clouds + 1], head[4 * num_clouds + 1:]
    pages = words[2 * nd:]
    M = int(cu[num_clouds])
    out = np.zeros((4, rows), dtype=np.int64)
    for t in range(rows):
        s = min(t, M - 1)
        c = max(i for i in range(num_clouds) if cu[i] <= s)
        r = s - cu[c]
        n_cur = n_prev[c] + cu[c + 1] - cu[c]
        pos = n_prev[c] + r
        out[:, t] = (pos, pages[table_off[c] + pos // P] * P + pos % P if t < M else scratch_row + t - M,
                     pair_off[c] + r * n_cur, c)
    return torch.from_numpy(out)


def _where(tables, P, ids, seqlens, n_prev):
    """Pure Python: node n_prev_c + r of cloud c sits at pool row table_c[pos // P] P + pos % P."""
    return [tables[c][(p + r) // P] * P + (p + r) % P for c, m, p in zip(ids, seqlens, n_prev) for r in range(m)]


def _random_step(g, P, clouds, rows_max):
    """A page book with `clouds` clouds (shared prefixes among them) and a step over a random subset."""
    book = PageTables(P)
    lens = {}
    for c in range(clouds):
        book.open(c)
        lens[c] = 0
        if c and g.random() < 0.4:                 # a fork of an earlier cloud
            src = int(g.integers(0, c))
            book.fork(src, c, lens[src])
            book.tables[c] = list(book.tables[c])
            lens[c] = lens[src]
        n = int(g.integers(1, 5000 if g.random() < 0.2 else 60))
        step = book.plan([c], [lens[c]], [n])
        book.commit(step, [c])
        lens[c] += n
    ids = list(g.permutation(clouds)[:int(g.integers(1, min(clouds, rows_max) + 1))])
    seqlens = [int(v) for v in g.integers(1, 4, len(ids))]
    while sum(seqlens) > rows_max:
        seqlens[int(np.argmax(seqlens))] -= 1
    n_prev = [lens[c] for c in ids]
    book.commit(book.plan(ids, n_prev, seqlens), ids)
    return book, ids, seqlens, n_prev


@pytest.mark.parametrize('P', [1, 7, 16])
@pytest.mark.parametrize('seed', range(4))
def test_descriptor_places_every_row_as_the_eager_step_does(P, seed):
    g = np.random.default_rng(seed)
    book, ids, seqlens, n_prev = _random_step(g, P, clouds=int(g.integers(1, 9)), rows_max=DECODE_GRAPH_ROWS)
    M = sum(seqlens)
    rows = 1 << (M - 1).bit_length()
    n_cur = [p + m for p, m in zip(n_prev, seqlens)]
    tables = [book.tables[c][:-(-n // P)] for c, n in zip(ids, n_cur)]
    desc = torch.zeros(ops.decode_desc_words(rows, rows * max(len(t) for t in tables)), dtype=torch.int32)
    assert ops.fill_decode_desc(desc, rows, n_prev, seqlens, [16] * len(ids), tables) == M
    scratch = 10 ** 6
    plan = host_plan(desc, rows, rows, P, scratch)
    # where _step and _where put each new row: its position, its pool row and its pair row
    dec = types.SimpleNamespace(page_size=P, _book=book)
    pos = torch.tensor([p + r for p, m in zip(n_prev, seqlens) for r in range(m)])
    lens = torch.tensor(seqlens)
    assert plan[1, :M].tolist() == _where(book.tables, P, ids, seqlens, n_prev) == \
        PagedCausalDecoder._where(dec, ids, lens, pos).tolist()
    assert plan[0, :M].tolist() == pos.tolist()
    pair_off = np.cumsum([0] + [m * n for m, n in zip(seqlens, n_cur)])[:-1]
    assert plan[2, :M].tolist() == [int(pair_off[i]) + r * n_cur[i] for i, m in enumerate(seqlens) for r in range(m)]
    assert plan[3, :M].tolist() == [i for i, m in enumerate(seqlens) for _ in range(m)]
    # padding rows repeat the last row and store into distinct scratch rows
    for t in range(M, rows):
        assert plan[[0, 2, 3], t].tolist() == plan[[0, 2, 3], M - 1].tolist()
        assert plan[1, t] == scratch + t - M


def test_descriptor_layout_and_room():
    tables = [[3, 1], [0]]
    desc = torch.full((ops.decode_desc_words(4, 5),), -7, dtype=torch.int32)
    assert ops.fill_decode_desc(desc, 4, [5, 2], [2, 1], [4, 2], tables) == 3
    head = desc[:2 * 21].view(torch.int64).tolist()
    assert head[:5] == [0, 2, 3, 3, 3]                     # cu_rows; clouds past the step's are empty
    assert head[5:9] == [5, 2, 0, 0]                       # n_prev
    assert head[9:13] == [4, 2, 1, 1]                      # k
    assert head[13:17] == [0, 14, 0, 0]                    # pair_off: 2 rows x 7 nodes before cloud 1
    assert head[17:21] == [0, 2, 0, 0]                     # table_off
    assert desc[42:45].tolist() == [3, 1, 0]
    with pytest.raises(ValueError, match='room'):
        ops.fill_decode_desc(desc, 4, [5, 2], [2, 1], [4, 2], [[3, 1, 2, 4, 5, 6], [0]])
    with pytest.raises(ValueError):
        ops.fill_decode_desc(desc, 1, [5, 2], [2, 1], [4, 2], tables)


# ---- rollback of a step's pages -------------------------------------------------------------------------------------------
def test_rollback_restores_tables_counts_and_free_list():
    book = PageTables(4, max_pages=16)
    for c in (0, 1):
        book.open(c)
    book.commit(book.plan([0, 1], [0, 0], [10, 3]), [0, 1])
    book.fork(0, 2, 10)
    book.tables[2] = list(book.tables[2])
    book.close(1)
    before = ({c: list(t) for c, t in book.tables.items()}, list(book.refs), list(book.free), book.reserved)
    plan = book.plan([0, 2], [10, 10], [7, 1])             # both write the shared page 2: one copy on write, fresh pages
    copies = book.commit(plan, [0, 2])
    assert copies and sum(plan.fresh)
    book.rollback(plan, [0, 2], copies)
    assert ({c: list(t) for c, t in book.tables.items()}, book.refs, book.free, book.reserved) == before


# ---- the switch -----------------------------------------------------------------------------------------------------------
def test_switch_is_registered_and_overridable(monkeypatch):
    monkeypatch.delenv('SE3B200_NO_DECODE_GRAPHS', raising=False)
    assert 'no_decode_graphs' in switches.FIELDS
    assert switches.ENV['no_decode_graphs'] == 'SE3B200_NO_DECODE_GRAPHS'
    assert not switches.current().no_decode_graphs
    with switches.override(no_decode_graphs=True):
        assert switches.current().no_decode_graphs
    assert not switches.current().no_decode_graphs


def test_descriptor_room_is_the_need_rounded_up_within_the_bound():
    dec = types.SimpleNamespace(_book=types.SimpleNamespace(max_pages=5000))
    room = lambda need, rows: PagedCausalDecoder._desc_room(dec, need, rows)
    assert room(1, 1) == 1024 and room(1024, 8) == 1024 and room(1025, 8) == 2048 and room(3000, 1) == 4096
    assert room(4999, 1) == 5000 and room(9000, 2) == 10000        # never past rows x max_pages
