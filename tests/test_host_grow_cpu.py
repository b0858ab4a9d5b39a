"""CPU: a numpy restatement of the in-place block mover of mutable host indexes (host_move.cu, DESIGN.md 3.5 "Mutable host indexes").

The host array is re-laid in place in chunks of whole destination blocks, staged through two buffers, with the gathers (reads) and
write-backs (writes) as an explicit event schedule.  Under the ordering rule -- a chunk's write-back waits for its own gather and the
gathers of every earlier chunk -- every order the schedule allows equals the out-of-place re-layout, for growth (descending chunks,
new rows staged into their chunk) and for the remove's block shift (ascending chunks).  A schedule that lets a write-back wait only for
its own chunk's gather (one stream per buffer) can run it before an earlier chunk's gather, and then some pattern comes out wrong."""
import numpy as np
import pytest

ROWS = 32


def layout(lens):
    """Tightly packed blocks: first block of every list, total blocks."""
    nb = (np.asarray(lens, np.int64) + ROWS - 1) // ROWS
    return np.concatenate([[0], np.cumsum(nb)[:-1]]).astype(np.int64), int(nb.sum())


def first_changed_block(old_len, new_len):
    """dph_first_changed_block: a list's first block when it moved, else its old tail block when its length changed."""
    bo, _ = layout(old_len)
    bn, nb = layout(new_len)
    for l in range(len(new_len)):
        if bn[l] != bo[l]:
            return int(bn[l])
        if new_len[l] != old_len[l]:
            return int(bn[l] + min(new_len[l], old_len[l]) // ROWS)
    return nb


def make_array(lens, cap, rng):
    """Host array [cap, 32] of row tokens (> 0), padding rows 0, and each list's rows in order."""
    bo, nb = layout(lens)
    arr = np.zeros((cap, ROWS), np.int64)
    rows = []
    for l, n in enumerate(lens):
        r = rng.integers(1, 2**62, n)
        arr.reshape(-1)[bo[l] * ROWS:bo[l] * ROWS + n] = r
        rows.append(r)
    return arr, rows


def out_of_place(rows, old_len, new_len, new_rows, cap):
    """The definition: every list's first min(old, new) rows stay at their offset, its new rows follow; into a fresh array."""
    bn, _ = layout(new_len)
    out = np.zeros((cap, ROWS), np.int64)
    for l in range(len(new_len)):
        keep = rows[l][:min(old_len[l], new_len[l])]
        r = np.concatenate([keep, new_rows[l]]) if new_rows is not None else keep
        assert len(r) == new_len[l]
        out.reshape(-1)[bn[l] * ROWS:bn[l] * ROWS + len(r)] = r
    return out


def first_moved_block(old_len, new_len):
    """The remove's block shift (remove.cu): from the first list whose first block moves."""
    bo, _ = layout(old_len)
    bn, nb = layout(new_len)
    moved = np.flatnonzero(bn != bo)
    return int(bn[moved[0]]) if len(moved) else nb


def clear_tails(arr, old_len, new_len):
    """The remove's tail clear (before the shift, in place): rows [new_len, end of its block) of every shrunk list become padding."""
    bo, _ = layout(old_len)
    flat = arr.reshape(-1)
    for l, (o, n) in enumerate(zip(old_len, new_len)):
        if n < o:
            flat[bo[l] * ROWS + n:bo[l] * ROWS + min(o, -(-n // ROWS) * ROWS)] = 0


def chunks(d_first, nb, cb, grow):
    """Destination chunks [c0, c1) of whole blocks: descending from the end for growth, ascending from d_first for the shift."""
    n = (nb - d_first + cb - 1) // cb
    if grow:
        return [(max(d_first, nb - (i + 1) * cb), nb - i * cb) for i in range(n)]
    return [(d_first + i * cb, min(nb, d_first + (i + 1) * cb)) for i in range(n)]


def schedule(n, rule=True):
    """Event dependencies.  ('R', i): gather of chunk i into buffer i % 2 (+ its new rows); ('W', i): its write-back.
    rule=True (host_move.cu): one gather stream and one write-back stream; W_i waits on the event recorded after R_i, which the
    in-order gather stream makes the mark of R_0 .. R_i; R_i waits for W_{i-2} (buffer reuse).
    rule=False: one stream per buffer -- W_i waits only for its own R_i."""
    deps = {}
    for i in range(n):
        if rule:
            deps["R", i] = [("R", i - 1)] * (i >= 1) + [("W", i - 2)] * (i >= 2)
            deps["W", i] = [("R", j) for j in range(i + 1)] + [("W", i - 1)] * (i >= 1)
        else:
            deps["R", i] = [("W", i - 2)] * (i >= 2)
            deps["W", i] = [("R", i)]
    return deps


def orders(deps, rng, count):
    """`count` random topological orders of the events (every order the schedule allows can be drawn)."""
    for _ in range(count):
        done, order = set(), []
        while len(order) < len(deps):
            ready = sorted(e for e in deps if e not in done and all(d in done for d in deps[e]))
            e = ready[rng.integers(len(ready))]
            done.add(e)
            order.append(e)
        yield order


def move_in_place(arr, old_len, new_len, new_rows, cb, order_fn, rule=True):
    """Run the mover on a copy of arr under the given schedule (a shrink: after the remove's tail clear) -> (array, written block
    ranges, first destination block, the array as the mover found it)."""
    arr = arr.copy()
    grow = all(n >= o for n, o in zip(new_len, old_len))
    bo, _ = layout(old_len)
    bn, nb = layout(new_len)
    if not grow:
        clear_tails(arr, old_len, new_len)
    before = arr.copy()
    d_first = first_changed_block(old_len, new_len) if grow else first_moved_block(old_len, new_len)
    cs = chunks(d_first, nb, cb, grow)
    buf = [np.zeros((cb, ROWS), np.int64) for _ in range(2)]
    owner = np.repeat(np.arange(len(new_len)), (np.asarray(new_len) + ROWS - 1) // ROWS)     # list of every new block
    written = []
    for kind, i in order_fn(schedule(len(cs), rule)):
        c0, c1 = cs[i]
        b = buf[i % 2]
        if kind == "R":
            b[:] = 0
            for blk in range(c0, c1):
                l = owner[blk]
                k = blk - bn[l]
                if k < (old_len[l] + ROWS - 1) // ROWS:               # the same list's old block, whole; zeros past its old end
                    b[blk - c0] = arr[bo[l] + k]
            if new_rows is not None:                                   # stage the new rows that land in this chunk
                for l in range(len(new_len)):
                    for t, r in enumerate(new_rows[l]):
                        j = old_len[l] + t
                        blk = bn[l] + j // ROWS
                        if c0 <= blk < c1:
                            b[blk - c0, j % ROWS] = r
        else:
            arr[c0:c1] = b[:c1 - c0]
            written.append((c0, c1))
    return arr, written, d_first, before


def pattern(rng, nlist, grow, max_len=200, long_list=None):
    old = rng.integers(0, max_len, nlist) * (rng.random(nlist) < 0.8)
    if long_list is not None:
        old[long_list] = 9 * ROWS + 5
    if grow:
        delta = rng.integers(0, 70, nlist) * (rng.random(nlist) < 0.5)
        new = old + delta
    else:
        new = np.maximum(old - rng.integers(0, 70, nlist) * (rng.random(nlist) < 0.5), 0)
    return old.astype(np.int64), new.astype(np.int64)


def check(old, new, cb, rng, n_orders=4):
    cap = max(layout(old)[1], layout(new)[1]) + 3                      # spare capacity at the array's end
    arr, rows = make_array(old, cap, rng)
    grow = bool((new >= old).all())
    new_rows = [rng.integers(1, 2**62, int(n - o)) for n, o in zip(new, old)] if grow else None
    want = out_of_place(rows, old, new, new_rows, cap)
    _, nb = layout(new)
    start = first_changed_block(old, new) if grow else first_moved_block(old, new)
    for order in orders(schedule(len(chunks(start, nb, cb, grow))), rng, n_orders):
        got, written, d_first, before = move_in_place(arr, old, new, new_rows, cb, lambda deps: order)
        assert np.array_equal(got[:nb], want[:nb]), (old, new, cb)
        assert np.array_equal(got[:d_first], before[:d_first])       # the mover touches nothing below its first block
        assert sorted(written) == sorted(chunks(d_first, nb, cb, grow))
    return d_first, nb


@pytest.mark.parametrize("grow", [True, False])
@pytest.mark.parametrize("cb", [1, 2, 3, 7, 64])
def test_random_patterns_equal_the_out_of_place_relayout(grow, cb):
    rng = np.random.default_rng(cb * 2 + grow)
    for trial in range(30):
        nlist = int(rng.integers(1, 12))
        old, new = pattern(rng, nlist, grow, long_list=int(rng.integers(nlist)) if trial % 3 == 0 else None)
        check(old, new, cb, rng)


def test_a_list_longer_than_a_chunk_moves_through_several_chunks():
    rng = np.random.default_rng(1)
    old = np.array([40, 10 * ROWS + 3, 7, 0, 65], np.int64)
    new = old + np.array([1, 0, 30, 2, 0])
    d_first, nb = check(old, new, 3, rng, n_orders=20)
    assert d_first == 1 and nb - d_first > 3 * 3


def test_growth_at_list_zero_moves_everything():
    rng = np.random.default_rng(2)
    old = np.array([64, 33, 100, 5, 31], np.int64)
    new = old + np.array([1, 0, 0, 0, 0])
    d_first, nb = check(old, new, 2, rng, n_orders=20)
    assert d_first == 2 and layout(new)[0][1] == layout(old)[0][1] + 1     # every later list moves up one block


def test_growth_at_the_last_list_moves_nothing():
    rng = np.random.default_rng(3)
    old = np.array([64, 33, 100, 5, 40], np.int64)
    new = old + np.array([0, 0, 0, 0, 100])
    d_first, nb = check(old, new, 1, rng, n_orders=20)
    assert (layout(new)[0] == layout(old)[0]).all() and d_first == layout(old)[0][4] + 1    # from the old tail block of the last list


def test_a_chunk_of_one_block_and_nothing_to_move():
    rng = np.random.default_rng(4)
    for old, new in (([32, 10], [33, 10]), ([5, 0, 7], [5, 0, 8]), ([10, 20], [10, 20])):
        d_first, nb = check(np.array(old), np.array(new), 1, rng, n_orders=10)
    assert d_first == nb                                                # equal layouts: no chunk at all


def test_breaking_the_ordering_rule_gives_a_wrong_result():
    """One stream per buffer: chunk 1's write-back may run before chunk 0's gather, which reads a source in chunk 1's destinations."""
    rng = np.random.default_rng(5)
    old = np.array([ROWS, 3 * ROWS], np.int64)                          # list 1: old blocks 1..3
    new = np.array([ROWS + 1, 3 * ROWS], np.int64)                       # list 0 gains a block: list 1 moves to blocks 2..4
    cap = 6
    arr, rows = make_array(old, cap, rng)
    new_rows = [rng.integers(1, 2**62, 1), np.zeros(0, np.int64)]
    want = out_of_place(rows, old, new, new_rows, cap)
    bad_order = [("R", 1), ("W", 1), ("R", 0), ("W", 0), ("R", 2), ("W", 2), ("R", 3), ("W", 3)]
    deps = schedule(4, rule=False)
    assert all(all(bad_order.index(d) < bad_order.index(e) for d in deps[e]) for e in bad_order)    # allowed without the rule
    good_deps = schedule(4, rule=True)
    assert not all(all(bad_order.index(d) < bad_order.index(e) for d in good_deps[e]) for e in bad_order)   # forbidden by it
    got = move_in_place(arr, old, new, new_rows, 1, lambda d: bad_order, rule=False)[0]
    assert not np.array_equal(got[:5], want[:5])
    # and random patterns under random schedules without the rule come out wrong some of the time, never with it
    wrong = 0
    for trial in range(40):
        o, n = pattern(rng, int(rng.integers(2, 8)), trial % 2 == 0)
        cap = max(layout(o)[1], layout(n)[1])
        a, rs = make_array(o, cap, rng)
        nr = [rng.integers(1, 2**62, int(y - x)) for x, y in zip(o, n)] if (n >= o).all() else None
        w = out_of_place(rs, o, n, nr, cap)
        nb = layout(n)[1]                                                  # a shrink leaves stale blocks past the new end
        for rule in (True, False):
            g = move_in_place(a, o, n, nr, 1, lambda d: next(orders(d, rng, 1)), rule=rule)[0]
            if rule:
                assert np.array_equal(g[:nb], w[:nb])
            else:
                wrong += not np.array_equal(g[:nb], w[:nb])
    assert wrong > 0
