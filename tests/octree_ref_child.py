"""The compiled reference octree (oracle/_ref/svo/svo_ref.so, built by oracle/build_ref.py) in a child process, and the runner the
octree comparison tests use to start it.

Why a child process per tree:
- `Octant::next_index_` (the node id counter) is a process global.  Only the reference's four-argument constructor resets it, and
  `init` does not, so a process numbers the nodes of its first tree only from 0.  Its pickle's `__setstate__` calls that
  constructor, so a tree unpickled in a fresh process is numbered from 0 too.
- The product's TorchScript shim registers a class of the same name, `torch.classes.svo.Octree`.
So the child imports torch and numpy only and loads nothing but svo_ref.so.

    python octree_ref_child.py SVO_REF_SO CASE.npz OUT.npz [--save-after K --state STATE] [--restore STATE --first K]

builds one tree from the case file (tests/octree_cases.py, Case.arrays): `init(grid_dim, 16, voxel_size)`, then one `insert` per
batch, and after every batch i stores in OUT.npz:
  voxels{i} children{i} features{i}   get_centres_and_children()
  gv{i} lv{i}                         get_voxels(), get_leaf_voxels()
  counts{i}                           [count_nodes(), count_leaf_nodes()]
  try{i}                              try_insert(probe) for every probe batch, as float64
  has{i}                              has_voxel(point) for every point, as bool
`get_features` is bound but its body is empty with no return statement (octree.cpp:208-210), so calling it is undefined
behaviour; it is not called.  With --save-after K the tree is pickled after batch K into STATE.  With --restore the tree is
unpickled from STATE (the reference replays the pickled points), its state is stored as batch K, and batches K + 1.. follow."""
import os
import pickle
import subprocess
import sys

import numpy as np


def _dump(t, z, out, i):
    import torch
    v, c, f = t.get_centres_and_children()
    out[f"voxels{i}"], out[f"children{i}"], out[f"features{i}"] = v.numpy(), c.numpy(), f.numpy()
    out[f"gv{i}"] = t.get_voxels().numpy()
    out[f"lv{i}"] = t.get_leaf_voxels().numpy()
    out[f"counts{i}"] = np.array([t.count_nodes(), t.count_leaf_nodes()], np.int64)
    out[f"try{i}"] = np.array([t.try_insert(torch.from_numpy(z[f"probe{k}"])) for k in range(int(z["n_probes"]))], np.float64)
    out[f"has{i}"] = np.array([t.has_voxel(torch.from_numpy(np.ascontiguousarray(p))) for p in z["points"]], bool)


def child_main(argv):
    import torch
    so, case_path, out_path = argv[:3]
    opts = dict(zip(argv[3::2], argv[4::2]))
    torch.ops.load_library(so)
    z = np.load(case_path)
    out = {}
    if "--restore" in opts:
        with open(opts["--restore"], "rb") as fh:
            t = pickle.load(fh)
        first = int(opts["--first"])
        _dump(t, z, out, first)
        first += 1
    else:
        t = torch.classes.svo.Octree()
        t.init(int(z["grid_dim"]), 16, float(z["voxel_size"]))
        first = 0
    for i in range(first, int(z["n_batches"])):
        t.insert(torch.from_numpy(z[f"batch{i}"]))
        _dump(t, z, out, i)
        if opts.get("--save-after") == str(i):
            with open(opts["--state"], "wb") as fh:
                pickle.dump(t, fh)
    np.savez(out_path, **out)


# -- the runner ------------------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SVO_REF = os.path.join(ROOT, "oracle", "_ref", "svo", "svo_ref.so")


def _run(args, timeout=900):
    p = subprocess.run([sys.executable, os.path.abspath(__file__), SVO_REF, *args], capture_output=True, text=True, timeout=timeout)
    if p.returncode != 0:
        return f"reference child {' '.join(args)} exited with {p.returncode}:\n{p.stderr[-4000:]}"
    return None


def run_cases(cases, tmpdir, workers=None):
    """Runs the reference on every case (name -> octree_cases.Case) in child processes, `workers` at a time, and returns
    name -> (dump of the uninterrupted run, dump of the restored run or None, error message or None).  Every child has exited when
    this returns; the dumps are npz files under tmpdir."""
    from concurrent.futures import ThreadPoolExecutor

    def one(item):
        name, case = item
        cpath, out = os.path.join(tmpdir, f"{name}.case.npz"), os.path.join(tmpdir, f"{name}.ref.npz")
        np.savez(cpath, **case.arrays())
        if case.restore_after is None:
            return name, (out, None, _run([cpath, out]))
        state, out2 = os.path.join(tmpdir, f"{name}.state.pkl"), os.path.join(tmpdir, f"{name}.restored.npz")
        err = _run([cpath, out, "--save-after", str(case.restore_after), "--state", state])
        if err is None:
            err = _run([cpath, out2, "--restore", state, "--first", str(case.restore_after)])
        return name, (out, out2, err)

    with ThreadPoolExecutor(max_workers=workers or min(16, os.cpu_count() or 1)) as ex:
        return dict(ex.map(one, cases.items()))


def load(path):
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


# -- the comparison --------------------------------------------------------------------------------------------------------------
def _same(x, y, what):
    """Equal dtype, shape and bytes (so -0.0 differs from 0.0); on a mismatch the message names the first differing row."""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    assert x.dtype == y.dtype and x.shape == y.shape, f"{what}: {x.dtype}{list(x.shape)} vs the reference's {y.dtype}{list(y.shape)}"
    if x.tobytes() != y.tobytes():
        bad = np.argwhere((x != y) | (np.signbit(x) != np.signbit(y)) if x.dtype.kind == "f" else x != y)[0]
        raise AssertionError(f"{what}: differs at {tuple(bad)}: {x[tuple(bad[:1])]} vs the reference's {y[tuple(bad[:1])]}")


def glue(ref, i, voxel_size):
    """mapping.py:322-326 (update_grid_features) on the reference's get_centres_and_children after batch i: (centres, structure,
    vertex), the arrays the product's export_map returns."""
    import torch
    v, c, f = (torch.from_numpy(ref[f"{k}{i}"]) for k in ("voxels", "children", "features"))
    return ((v[:, :3] + v[:, -1:] / 2) * voxel_size).float(), torch.cat([c, v[:, -1:]], -1).int(), f


def glue_rows(features, vertex2row, n_rows):
    """mapping.py:294-317 (get_embeddings): the vertices of voxel_vertex_idx without a row, in their order in the flattened array,
    get rows n_rows, n_rows + 1, ...  The reference gives a vertex one row per reference to it and keeps one of them by a racy
    index_put_; the product gives it one row, numbered by its first reference (DESIGN.md section 5.2, deviation 4).  Returns
    vertex2row (-1 = no row) extended to the node count, and the new number of rows."""
    n = features.shape[0]
    v2r = np.full(n, -1, np.int32)
    v2r[:vertex2row.shape[0]] = vertex2row
    flat = features.reshape(-1)
    flat = flat[flat != -1]
    new = flat[v2r[flat] == -1]
    _, first = np.unique(new, return_index=True)
    order = new[np.sort(first)]
    v2r[order] = np.arange(n_rows, n_rows + order.shape[0], dtype=np.int32)
    return v2r, n_rows + order.shape[0]


def assert_equals_reference(tree, ref, i, case, where, probe_input=None):
    """Every output of `tree` (svo.Octree or svo.DeviceOctree) equals the reference's after batch i, exactly: the three arrays of
    get_centres_and_children, both counts, get_voxels, get_leaf_voxels, try_insert on every probe (as doubles), has_voxel on every
    point, and export_map equals the reference's glue.  probe_input maps a CPU int32 probe tensor to the tree's input (a device,
    say).  An empty probe is the one difference: the reference divides 0 by 0 (NaN), the product returns -1.0."""
    import torch
    at = f"{where}, after batch {i}"
    for k, x in zip(("voxels", "children", "features"), tree.get_centres_and_children()):
        _same(x.numpy(), ref[f"{k}{i}"], f"{at}: get_centres_and_children {k}")
    assert [tree.count_nodes(), tree.count_leaf_nodes()] == ref[f"counts{i}"].tolist(), f"{at}: count_nodes, count_leaf_nodes"
    _same(tree.get_voxels().numpy(), ref[f"gv{i}"], f"{at}: get_voxels")
    _same(tree.get_leaf_voxels().numpy(), ref[f"lv{i}"], f"{at}: get_leaf_voxels")
    conv = probe_input or (lambda t: t)
    tries = np.array([tree.try_insert(conv(torch.from_numpy(p))) for p in case.probes], np.float64)
    want = ref[f"try{i}"].copy()
    empty = np.array([p.shape[0] == 0 for p in case.probes], bool)
    assert np.isnan(want[empty]).all(), f"{at}: the reference's try_insert of an empty batch is no longer 0/0"
    want[empty] = -1.0
    _same(tries, want, f"{at}: try_insert")
    has = np.array([tree.has_voxel(p) for p in case.points], bool)
    _same(has, ref[f"has{i}"], f"{at}: has_voxel")
    for k, x, y in zip(("centres", "structure", "vertex"), tree.export_map(), glue(ref, i, case.voxel_size)):
        _same(x.numpy(), y.numpy(), f"{at}: export_map {k} against mapping.py:322-326 on the reference's arrays")


if __name__ == "__main__":
    child_main(sys.argv[1:])
