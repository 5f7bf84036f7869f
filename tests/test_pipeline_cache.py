"""InferencePipeline's graph cache without a GPU: _cached keeps the most recently used entry last, evicts the least
recently used ones at max_graphs, and replaces an entry its `fits` rejects at the same key."""
import collections
import itertools


def _pipe(max_graphs):
    from det3d_b200.apis import InferencePipeline
    pipe = object.__new__(InferencePipeline)          # the cache needs only _graphs and max_graphs
    pipe._graphs = collections.OrderedDict()
    pipe.max_graphs = max_graphs
    return pipe


def test_lookups_keep_the_most_recently_used_last():
    pipe, made = _pipe(4), itertools.count()
    entries = {k: pipe._cached(k, lambda: next(made)) for k in ("a", "b", "c")}
    assert list(pipe._graphs) == ["a", "b", "c"] and list(entries.values()) == [0, 1, 2]
    assert pipe._cached("a", lambda: next(made)) == 0                # a hit makes nothing
    assert list(pipe._graphs) == ["b", "c", "a"]
    assert pipe._cached("b", lambda: next(made), fits=lambda e: e == 1) == 1
    assert list(pipe._graphs) == ["c", "a", "b"] and next(made) == 3


def test_a_full_cache_evicts_the_least_recently_used():
    pipe, made = _pipe(3), itertools.count()
    for k in ("a", "b", "c"):
        pipe._cached(k, lambda: next(made))
    pipe._cached("a", lambda: next(made))
    assert pipe._cached("d", lambda: next(made)) == 3
    assert list(pipe._graphs) == ["c", "a", "d"]                    # b was the least recently used
    pipe._cached("e", lambda: next(made))
    assert list(pipe._graphs) == ["a", "d", "e"]
    pipe.max_graphs = 1                                             # evicts until there is room for one
    assert pipe._cached("f", lambda: next(made)) == 5
    assert list(pipe._graphs) == ["f"]


def test_an_entry_that_does_not_fit_is_replaced_at_its_key():
    pipe, made = _pipe(3), itertools.count()
    for k in ("a", "b", "c"):
        pipe._cached(k, lambda: next(made))
    assert pipe._cached("a", lambda: next(made), fits=lambda e: e != 0) == 3
    assert list(pipe._graphs) == ["b", "c", "a"]                    # full, yet no other entry was evicted
    assert pipe._graphs == {"a": 3, "b": 1, "c": 2}
    assert pipe._cached("a", lambda: next(made), fits=lambda e: e == 3) == 3
