"""CPU-only: map checkpoints (MapUpdater.state_dict / from_state_dict) and the node-array restore of the host tree.
  * nl_octree_nodes -> nl_octree_restore gives a tree whose every export, query and count equals the original's, and which
    continues like it after further inserts, at grid_dim 8, 64, 2^18 and 2^20; restored trees pickle as node arrays and continue;
  * a map saved after scan k and restored continues exactly like the uninterrupted map (state_dict and map_states after every
    later scan), with and without init_std, through torch.save / torch.load(weights_only=True);
  * every NL_TREE_* check rejects a hand-made mutation with exactly its bit, without touching the tree, and the new entry points
    reject bad arguments before any CUDA call.
"""
import copy
import io
import pickle

import numpy as np
import pytest
import torch

from test_device_octree_queries_cpu import _trees

ROOT, RANGE, LINK, PARENTS, SHAPE, ROWS, VERTICES = (1 << i for i in range(7))


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


def _host(nl, gd, batches):
    o = nl.svo.Octree()
    o.init(gd, 16, 0.3)
    for b in batches:
        o.insert(torch.from_numpy(b))
    return o


def _everything(o, queries):
    tensors = [*o.get_centres_and_children(), o.get_voxels(), o.get_leaf_voxels(), *o.export_map(), *o.export_nodes()]
    scalars = [o.count_nodes(), o.count_leaf_nodes(), o.count_export_nodes()] + [o.has_voxel(q[0]) for q in queries] + \
        [o.try_insert(torch.from_numpy(q)) for q in queries]
    return tensors, scalars


def _assert_same(a, b):
    assert a[1] == b[1]
    assert len(a[0]) == len(b[0])
    for x, y in zip(a[0], b[0]):
        assert x.dtype == y.dtype and torch.equal(x, y)


def _assert_same_dirty(a, b):
    for x, y in zip(a.export_dirty(), b.export_dirty()):
        assert x.dtype == y.dtype and np.array_equal(x, y)


@pytest.mark.parametrize("grid_dim", [8, 64, 1 << 18, 1 << 20])
def test_restored_host_tree_equals_the_original_and_continues(nl, grid_dim):
    batches = _trees()[grid_dim]
    queries = [np.ascontiguousarray(b[:50]) for b in batches] + [np.ascontiguousarray(batches[0][:20] + 1)]
    orig = _host(nl, grid_dim, batches[:1])
    orig.export_dirty()                                                 # a map update applied the first batch
    child, code, type_, level = orig.export_nodes()
    assert child.dtype == torch.int32 and code.dtype == torch.int64 and type_.dtype == torch.int8 and level.dtype == torch.uint8
    assert torch.equal(torch.from_numpy(grid_dim >> level.numpy().astype(np.int64)).float(),
                       torch.from_numpy(np.where(type_.numpy() == 1, 1, orig.get_centres_and_children()[0][:, 3].numpy()).astype(np.float32)))
    rest = nl.svo.Octree()
    rest.init(grid_dim, 16, 0.3)
    rest.load_nodes(child, code, type_, level)
    _assert_same(_everything(rest, queries), _everything(orig, queries))
    assert rest.export_dirty()[0].shape[0] == 0                         # nothing dirty
    for b in batches[1:] + [batches[0]]:                                # later batches, then a repeated one (seen points are a cache)
        orig.insert(torch.from_numpy(b))
        rest.insert(torch.from_numpy(b))
        _assert_same_dirty(rest, orig)
        _assert_same(_everything(rest, queries), _everything(orig, queries))
    again = pickle.loads(pickle.dumps(rest))                            # node-array pickle: no point history to replay
    assert "nodes" in rest.__getstate__() and "all_pts" in orig.__getstate__()
    deep = copy.deepcopy(rest)
    extra = np.ascontiguousarray(batches[-1][::-1] // 2)
    for t in (orig, again, deep):
        t.export_dirty()
        t.insert(torch.from_numpy(extra))
    _assert_same_dirty(again, orig)
    _assert_same(_everything(again, queries), _everything(orig, queries))
    _assert_same(_everything(deep, queries), _everything(orig, queries))


# -- checkpoints of a MapUpdater --------------------------------------------------------------------------------------------------
def _scans(nl, k=5):
    syn = nl.synthetic
    return [syn.make_scan(n_beams=16, n_az=160, seed=300 + i, sensor_xyz=(0.8 * i, 0.1 * i, 0.0)) for i in range(k)]


def _assert_same_state(a, b):
    assert set(a) == set(b)
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k
        else:
            assert type(a[k]) is type(b[k]) and a[k] == b[k], k


def _assert_same_map_states(a, b):
    assert set(a) == set(b)
    for k in a:
        if k == "_mapstate":
            for f in ("centres", "structure", "vox2row", "emb"):
                assert torch.equal(getattr(a[k], f), getattr(b[k], f)), f
        else:
            assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("init_std", [0.0, 0.01])
@pytest.mark.parametrize("k", [1, 3])
def test_saved_map_continues_like_the_uninterrupted_one(nl, init_std, k):
    scans = _scans(nl)
    mu = nl.mapping.MapUpdater(0.3, device="cpu", incremental=False, init_std=init_std, seed=7)
    for pts, _, pose in scans[:k]:
        mu.create_voxels(pts, pose)
    sd = mu.state_dict()
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    loaded = torch.load(buf, weights_only=True)
    _assert_same_state(loaded, sd)
    res = nl.mapping.MapUpdater.from_state_dict(loaded, device="cpu")
    _assert_same_state(res.state_dict(), sd)
    _assert_same_map_states(res.map_states, mu.map_states)
    assert res.generation == mu.generation and res.n_rows == mu.n_rows and np.array_equal(res.vertex2row, mu.vertex2row)
    with torch.no_grad():                                               # training changes the table between updates
        mu.embeddings.add_(0.125)
        res.embeddings.add_(0.125)
    for pts, _, pose in scans[k:]:
        mu.create_voxels(pts, pose)
        res.create_voxels(pts, pose)
        _assert_same_state(res.state_dict(), mu.state_dict())
        _assert_same_map_states(res.map_states, mu.map_states)
    assert "nodes" in res.svo.__getstate__()


def test_state_dict_refuses_inserts_not_applied_yet(nl):
    (pts, _, pose), (pts2, _, pose2) = _scans(nl, 2)
    mu = nl.mapping.MapUpdater(0.3, device="cpu", incremental=False)
    with pytest.raises(nl._capi.NerfLoamError, match="not applied"):
        mu.state_dict()                                                 # the root alone, never applied
    mu.create_voxels(pts, pose)
    mu.state_dict()
    mu.svo.insert(torch.from_numpy(nl.synthetic.voxelize(pts2, pose2, 0.3)))
    with pytest.raises(nl._capi.NerfLoamError, match="not applied"):
        mu.state_dict()
    mu.update_grid_features()
    mu.state_dict()


# -- the checks ---------------------------------------------------------------------------------------------------------------
def _state(nl):
    mu = nl.mapping.MapUpdater(1.0, grid_dim=64, device="cpu", incremental=False)
    rng = np.random.default_rng(4)
    for n in (30, 200):
        mu.insert_voxels(torch.from_numpy(rng.integers(0, 63, (n, 3)).astype(np.int32)))
    return mu.state_dict()


def _find(sd, mutate, want, nl):
    """The first candidate mutation whose verdict is exactly `want`, as a mutated copy of sd."""
    for cand in mutate(sd):
        if _bits(nl, cand) == want:
            return cand
    raise AssertionError("no candidate mutation with exactly the wanted bit")


def _bits(nl, s):
    return nl.svo.validate_nodes(s["grid_dim"], s["child"], s["code"], s["type"], s["level"], s["vertex2row"], s["embeddings"].shape[0])


def _copy(sd):
    return {k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in sd.items()}


def _empty_tree(sd):
    s = _copy(sd)
    for k in ("child", "code", "type", "level", "vertex2row"):
        s[k] = s[k][:0].clone()
    s["embeddings"] = s["embeddings"][:0].clone()
    yield s


def _each(sd, nodes, edit):
    for i in nodes:
        s = _copy(sd)
        if edit(s, int(i)) is not False:
            yield s


def _mutations(sd):
    """check -> candidate generators; each check's mutation must produce exactly its bit."""
    t, lv, ch = sd["type"].numpy(), sd["level"].numpy(), sd["child"].numpy()
    L = int(lv.max())
    n = t.shape[0]
    nonleaf_with_gap = [i for i in range(n) if t[i] == -1 and (ch[i] == -1).any()]
    feature = np.nonzero(t == 1)[0]
    surface = np.nonzero(t == 0)[0]
    level_below = np.nonzero((t == -1) & (lv == L - 1))[0]
    multi = [i for i in range(n) if t[i] == -1 and (ch[i] >= 0).sum() >= 2]

    def gap(s, i, value):
        s["child"][i, int(np.nonzero(s["child"][i].numpy() == -1)[0][0])] = value(i)

    def set_(k, v):
        def f(s, i):
            s[k][i] = v
        return f

    def drop_child(s, i):
        s["child"][i, int(np.nonzero(s["child"][i].numpy() >= 0)[0][0])] = -1

    def first_row_out(s, i):
        v = int(np.nonzero(s["vertex2row"].numpy() >= 0)[0][0])
        s["vertex2row"][v] = s["embeddings"].shape[0]

    def share_row(s, i):
        v = np.nonzero(s["vertex2row"].numpy() >= 0)[0]
        s["vertex2row"][v[1]] = s["vertex2row"][v[0]]

    def low_bits(s, i):
        s["code"][i] |= 1

    return {
        ROOT: [_empty_tree(sd)],
        RANGE: [_each(sd, nonleaf_with_gap[:1], lambda s, i: gap(s, i, lambda i: n)), _each(sd, nonleaf_with_gap[1:2], lambda s, i: gap(s, i, lambda i: i)),
                _each(sd, feature[:5], set_("type", 5))],
        LINK: [_each(sd, level_below[:5], low_bits)],
        PARENTS: [_each(sd, multi[:5], drop_child)],
        SHAPE: [_each(sd, feature[:5], set_("type", -1)), _each(sd, level_below[:5], set_("type", 0))],
        ROWS: [_each(sd, [0], first_row_out), _each(sd, [0], share_row)],
        VERTICES: [_each(sd, surface, set_("type", 1)), _each(sd, feature, set_("type", 0))],
    }


def mutated_states(nl):
    """(bit, mutated state) pairs, at least one per check and per mutation kind (shared with the GPU test)."""
    sd = _state(nl)
    assert _bits(nl, sd) == 0
    out = []
    for bit, gens in _mutations(sd).items():
        for g in gens:
            out.append((bit, _find(sd, lambda _: g, bit, nl)))
    return sd, out


def test_each_check_rejects_its_mutation_with_exactly_its_bit(nl):
    sd, cases = mutated_states(nl)
    assert {b for b, _ in cases} == {ROOT, RANGE, LINK, PARENTS, SHAPE, ROWS, VERTICES} and len(cases) >= 12
    tree = nl.svo.Octree()
    tree.init(64, 16, 1.0)
    tree.load_nodes(sd["child"], sd["code"], sd["type"], sd["level"])
    before = tree.export_nodes()
    for bit, s in cases:
        name = nl._capi.tree_checks_failed(bit)[0]
        assert _bits(nl, s) == bit
        with pytest.raises(nl._capi.NerfLoamError, match=f"failed checks: {name}$"):
            nl.mapping.MapUpdater.from_state_dict(s, device="cpu")
        structural = nl.svo.validate_nodes(64, s["child"], s["code"], s["type"], s["level"])
        assert structural == (bit if bit < ROWS else 0)
        if structural:
            with pytest.raises(nl._capi.NerfLoamError, match=name):
                tree.load_nodes(s["child"], s["code"], s["type"], s["level"])
            for x, y in zip(tree.export_nodes(), before):                # untouched
                assert torch.equal(x, y)
    # a structurally broken tree is not walked: its rows are not checked
    s = _copy(sd)
    s["vertex2row"][:] = -5
    s["type"][0] = 7
    assert _bits(nl, s) == ROOT | RANGE


def test_from_state_dict_checks_the_format_before_the_tree(nl):
    sd = _state(nl)
    bad = {
        "format": ("format", 2), "grid_dim": ("grid_dim", 100), "grid_dim ": ("grid_dim", 1 << 21), "embed_dim": ("embed_dim", 8),
        "child": ("child", sd["child"].long()), "code": ("code", sd["code"].float()), "level": ("level", sd["level"][:-1]),
        "embeddings": ("embeddings", sd["embeddings"].float()), "embeddings ": ("embeddings", sd["embeddings"][:, :8]),
        "vertex2row": ("vertex2row", sd["vertex2row"][:5]),
    }
    for name, (k, v) in bad.items():
        s = _copy(sd)
        s[k] = v
        with pytest.raises(nl._capi.NerfLoamError, match="malformed checkpoint.*" + name.strip()):
            nl.mapping.MapUpdater.from_state_dict(s, device="cpu")
    s = _copy(sd)
    del s["level"]
    with pytest.raises(nl._capi.NerfLoamError, match="keys level"):
        nl.mapping.MapUpdater.from_state_dict(s, device="cpu")


def test_new_entry_points_reject_bad_arguments_without_touching_the_gpu(nl):
    L = nl._capi.lib()
    err = lambda: L.nl_last_error().decode()
    one = 16                                                              # a non-null stand-in pointer; never dereferenced
    assert L.nl_octree_validate(100, 1, one, one, one, one, None, 0) < 0 and "grid_dim" in err()
    assert L.nl_octree_validate(64, -1, one, one, one, one, None, 0) < 0 and "sizes" in err()
    assert L.nl_octree_validate(64, 1, one, one, one, one, None, -1) < 0 and "sizes" in err()
    for i in range(4):
        args = [one] * 4
        args[i] = None
        assert L.nl_octree_validate(64, 3, *args, None, 0) < 0 and "null" in err()
    assert L.nl_octree_validate(64, 0, None, None, None, None, None, 0) == ROOT
    assert L.nl_octree_nodes(None, one, one, one, one) < 0 and "null" in err()
    t = nl.svo.Octree()
    t.init(64, 16, 1.0)
    for i in range(4):
        args = [one] * 4
        args[i] = None
        assert L.nl_octree_nodes(t._h, *args) < 0 and "null" in err()
        assert L.nl_octree_restore(t._h, *args, 3) < 0 and "null" in err()
    assert L.nl_octree_restore(None, one, one, one, one, 3) < 0 and "bad" in err()
    assert L.nl_octree_restore(t._h, one, one, one, one, -1) < 0 and "bad" in err()
    assert L.nl_octree_restore(t._h, None, None, None, None, 0) == ROOT and t.count_nodes() == 1
    big = 1 << 30
    val = lambda gd, n, arrays, v2r, n_rows, ws, wsb, out: L.nl_devoctree_validate(gd, n, *arrays, v2r, n_rows, ws, wsb, out, None)
    assert val(6, 10, [one] * 4, None, 0, 256, big, one) != 0 and "grid_dim" in err()
    assert val(1 << 21, 10, [one] * 4, None, 0, 256, big, one) != 0 and "grid_dim" in err()
    assert val(64, -1, [one] * 4, None, 0, 256, big, one) != 0 and "sizes" in err()
    assert val(64, 1 << 31, [one] * 4, None, 0, 256, big, one) != 0 and "sizes" in err()
    assert val(64, 10, [one] * 4, one, -1, 256, big, one) != 0 and "sizes" in err()
    assert val(64, 10, [one] * 4, None, 0, 256, big, None) != 0 and "null" in err()
    assert val(64, 10, [one] * 4, None, 0, None, big, one) != 0 and "null" in err()
    for i in range(4):
        args = [one] * 4
        args[i] = None
        assert val(64, 10, args, None, 0, 256, big, one) != 0 and "null" in err()
    assert val(64, 1000, [one] * 4, None, 0, 256, 16, one) != 0 and "workspace of 16 bytes" in err()
    assert val(64, 10, [one] * 4, None, 0, 16, big, one) != 0 and "aligned" in err()
