"""Mirror of the reference's ``postprocessing/clean_smallparts.py``: removes the small and stray ("flying") parts from
the meshes ``create_sdf`` writes, before the evaluation scripts read them.  Same functions, arguments and file naming
(``separate_single_mesh``, ``clean_single_mesh``, ``clean_meshes``, ``build_file_dict``); the component labelling, the
per-component reductions and the compaction run on the GPU (Engine.load_mesh + Engine.clean_mesh) instead of PyMesh.

    python -m disn_b200.clean_smallparts --src_dir <test_objs/65_0.0> --tar_dir <test_objs/65_0.0_clean> [--thread_n 10]

cleans every ``<src_dir>/<cat_id>/*.obj`` into ``<tar_dir>/<cat_id>/`` with the reference's thresholds (0.5 / 0.3).
One Engine serves all threads, serialised by a lock (a context is not thread-safe); OBJ parsing and writing run on the
worker threads.
"""
from __future__ import annotations

import argparse
import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .create_sdf import read_obj, write_obj

_ENGINE = None
_LOCK = threading.Lock()


def _engine():
    global _ENGINE
    if _ENGINE is None:
        from .engine import Engine
        _ENGINE = Engine(device=0, precision="fp32")
    return _ENGINE


def separate_single_mesh(src_mesh, tar_mesh):
    """clean_smallparts.py:27-36: write the mesh to tar_mesh + ".obj" and each component to tar_mesh + "_<i>.obj"
    (components in order of their smallest face; each with the vertices its faces reference, in their original order)."""
    verts, faces = read_obj(src_mesh)
    with _LOCK:
        eng = _engine()
        eng.load_mesh(verts, faces)
        counts, labels = eng.clean_mesh(np.inf, -1.0, fetch=False, want_labels=True)   # keeps every component
    write_obj(tar_mesh + ".obj", verts, faces)
    for count in range(counts.n_components):
        f = faces[labels == count]
        used = np.zeros(len(verts), bool)
        used[f.reshape(-1)] = True
        vmap = np.cumsum(used) - used
        print("dis_mesh.vertices.shape", (int(used.sum()), 3))
        print("dis_mesh.faces.shape", f.shape)
        write_obj(tar_mesh + "_" + str(count) + ".obj", verts[used], vmap[f])


def clean_single_mesh(src_mesh, tar_mesh, dist_thresh, num_thresh):
    """clean_smallparts.py:38-54: keep the components with more than max_count * num_thresh vertices whose centroid lies
    closer than dist_thresh to the origin, and write them to tar_mesh."""
    verts, faces = read_obj(src_mesh)
    with _LOCK:
        eng = _engine()
        eng.load_mesh(verts, faces)
        verts, faces = eng.clean_mesh(dist_thresh, num_thresh)
    write_obj(tar_mesh, verts, faces)
    print("threshes:", str(dist_thresh), str(num_thresh), " clean: ", src_mesh, " create: ", tar_mesh)


def clean_meshes(cats, src_dir, tar_dir, dist_thresh=0.5, num_thresh=0.3, thread_n=12):
    """clean_smallparts.py:56-70: cats maps a category name to its directory (cat_id) under src_dir / tar_dir."""
    for cat_nm, cat_id in cats.items():
        src_cat_dir = os.path.join(src_dir, cat_id)
        tar_cat_dir = os.path.join(tar_dir, cat_id)
        os.makedirs(tar_cat_dir, exist_ok=True)
        _, _, src_file_lst, tar_file_lst = build_file_dict(src_cat_dir, tar_cat_dir)
        with ThreadPoolExecutor(max_workers=max(1, thread_n)) as ex:
            for fut in [ex.submit(clean_single_mesh, s, t, dist_thresh, num_thresh)
                        for s, t in zip(src_file_lst, tar_file_lst)]:
                fut.result()
        print("done with ", cat_nm, cat_id)
    print("done!")


def build_file_dict(src_dir, tar_dir):
    """clean_smallparts.py:72-93: files of src_dir grouped by object id (the second `_`-separated field of the name,
    <cat_id>_<obj_id>_<view>.obj) -> (src_file_dict, tar_file_dict, src_file_lst, tar_file_lst)."""
    src_file_dict, tar_file_dict = {}, {}
    src_file_lst, tar_file_lst = [], []
    for file in os.listdir(src_dir):
        src_full_path = os.path.join(src_dir, file)
        tar_full_path = os.path.join(tar_dir, file)
        if os.path.isfile(src_full_path):
            obj_id = file.split("_")[1]
            src_file_dict.setdefault(obj_id, []).append(src_full_path)
            src_file_lst.append(src_full_path)
            tar_file_dict.setdefault(obj_id, []).append(tar_full_path)
            tar_file_lst.append(tar_full_path)
    return src_file_dict, tar_file_dict, src_file_lst, tar_file_lst


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--src_dir", type=str, default="", help="src directory, before clean")
    parser.add_argument("--tar_dir", type=str, default="", help="where to store")
    parser.add_argument("--thread_n", type=int, default=10, help="parallelism")
    flags = parser.parse_args(argv)
    print(flags)
    # every category directory present under src_dir (the reference hard-codes a category dict)
    cats = {d: d for d in sorted(os.listdir(flags.src_dir)) if os.path.isdir(os.path.join(flags.src_dir, d))}
    clean_meshes(cats, flags.src_dir, flags.tar_dir, dist_thresh=0.5, num_thresh=0.3, thread_n=flags.thread_n)


if __name__ == "__main__":
    main()
