"""Host-side logic of the round-2 fast paths that needs no GPU: the lazily materialised meta dict of rasterization()
and the capacity prediction of the intersection stage."""
from gsplat_b200 import ops
from gsplat_b200.rendering import _Lazy, _Meta


def test_meta_resolves_lazy_values_on_every_read_path():
    calls = []

    def make():
        calls.append(1)
        return "ids"

    m = _Meta({"a": 1, "isect_ids": _Lazy(make)})
    assert "isect_ids" in m and len(m) == 2 and calls == []  # membership / size do not materialise
    assert m["a"] == 1 and calls == []
    assert m["isect_ids"] == "ids" and m["isect_ids"] == "ids" and calls == [1]  # computed once, then stored
    for read in (lambda d: dict(d), lambda d: {**d}, lambda d: dict(d.items()), lambda d: d.copy(), lambda d: {k: d[k] for k in d}):
        m = _Meta({"a": 1, "isect_ids": _Lazy(lambda: "ids")})
        assert read(m) == {"a": 1, "isect_ids": "ids"}
    m = _Meta({"isect_ids": _Lazy(lambda: "ids")})
    assert m.get("isect_ids") == "ids" and m.get("missing", 7) == 7
    m = _Meta({"isect_ids": _Lazy(lambda: "ids")})
    assert list(m.values()) == ["ids"]
    m = _Meta({"isect_ids": _Lazy(lambda: "ids")})
    assert m.pop("isect_ids") == "ids" and m.pop("isect_ids", None) is None


def _predictor():
    p = object.__new__(ops._IsectPredictor)  # the constructor allocates pinned memory / a stream: not needed here
    p.hist, p.hits, p.misses = [], 0, 0
    return p


def test_isect_capacity_prediction():
    p = _predictor()
    assert p.capacities(1000) is None  # nothing seen yet: the first call of a shape reads the totals first
    p.observe(100000, 5000, 40)
    cap_vis, cap_isects, max_tiles = p.capacities(10**6)
    assert cap_vis >= 5000 and cap_isects >= 100000 and max_tiles == 40
    assert cap_vis <= 5000 * 1.04 + 512 and cap_isects <= 100000 * 1.04 + 2048  # a few percent of padding, not more
    assert p.capacities(5100)[0] == 5100  # never more rows than exist
    # the capacities follow the maximum of the last eight calls (views of a trainer differ) and forget older ones
    p.observe(300000, 9000, 200)
    assert p.capacities(10**6)[1] >= 300000 and p.capacities(10**6)[2] == 200
    for _ in range(8):
        p.observe(50000, 2000, 10)
    cap_vis, cap_isects, max_tiles = p.capacities(10**6)
    assert cap_isects < 60000 and cap_vis < 3000 and max_tiles == 10
    # an empty view must not produce zero-sized speculative launches
    q = _predictor()
    q.observe(0, 0, 0)
    assert q.capacities(1000) is None


def test_capacity_padding_model():
    """numpy model of the capacity-sized intersection stage (isect.cu: gsb200_isect_sorted): padding pairs carry the largest
    key and sit behind the real pairs, the stable sort only looks at the low `end_bit` bits, and the offsets kernel reads the
    first totals[0] sorted keys -- the result must equal the exact pipeline's, also when the number of (image, tile) cells is a
    power of two (the padding key then aliases the last real cell) and when a miss leaves garbage keys in the list."""
    import numpy as np

    def offsets_of(sorted_keys, n_real, total_tiles):
        off = np.zeros(total_tiles, np.int64)
        for s in range(n_real):  # isect_offsets_tilekeys_kernel, one iteration per thread
            ident = min(int(sorted_keys[s]), total_tiles - 1)
            prev = int(sorted_keys[s - 1]) if s > 0 else -1
            off[prev + 1 : ident + 1] = s
            if s == n_real - 1:
                off[ident + 1 :] = n_real
        return off

    rng = np.random.RandomState(3)
    for total_tiles in (4096, 2800, 1):
        end_bit = max(1, int(total_tiles - 1).bit_length())
        n_real, cap = 5000, 5600
        keys = rng.randint(0, total_tiles, n_real).astype(np.uint16)
        rows = np.arange(n_real, dtype=np.int32)  # emission order = depth order
        padded = np.concatenate([keys, np.full(cap - n_real, 0xFFFF, np.uint16)])
        prow = np.concatenate([rows, np.zeros(cap - n_real, np.int32)])
        order = np.argsort(padded & ((1 << end_bit) - 1), kind="stable")  # LSD radix sort on bits [0, end_bit)
        exact = np.argsort(keys, kind="stable")
        assert np.array_equal(prow[order][:n_real], rows[exact]) and np.array_equal(padded[order][:n_real], keys[exact])
        want = np.searchsorted(keys[exact], np.arange(total_tiles), side="left")
        assert np.array_equal(offsets_of(padded[order], n_real, total_tiles), want)
    # after a miss some slots hold uninitialised keys: every write must still land inside the array
    garbage = rng.randint(0, 65536, 300).astype(np.uint16)
    off = offsets_of(garbage, 300, 2800)
    assert off.shape == (2800,) and off.min() >= 0 and off.max() <= 300
