"""What the three evaluation drivers (eval_cd_emd, eval_f_score, eval_iou) share: the reference scripts' category dicts
(test/test_cd_emd.py:319-344, test/test_f_score.py:262-287, test/test_iou.py:241-267) and the file listing.

The reference lists a results directory with os.listdir, whose order is the file system's; random.sample and the
view order then depend on it.  The drivers list in sorted order, so that the same seeds draw the same views on every
file system (the reference's draws on a file system that lists in sorted order).
"""
from __future__ import annotations

import os

from .create_sdf import read_obj

CATS_ALL = {
    "watercraft": "04530566",
    "rifle": "04090263",
    "display": "03211117",
    "lamp": "03636649",
    "speaker": "03691459",
    "chair": "03001627",
    "bench": "02828884",
    "cabinet": "02933112",
    "car": "02958343",
    "airplane": "02691156",
    "sofa": "04256520",
    "table": "04379243",
    "phone": "04401088",
}
# "clean" in test_cd_emd.py / test_f_score.py
CATS_CLEAN = {"cabinet": "02933112", "display": "03211117", "speaker": "03691459", "rifle": "04090263",
              "watercraft": "04530566"}
# "clean" in test_iou.py (also lamp)
CATS_CLEAN_IOU = {"cabinet": "02933112", "display": "03211117", "lamp": "03636649", "speaker": "03691459",
                  "rifle": "04090263", "watercraft": "04530566"}


def select_cats(category: str, clean=CATS_CLEAN) -> dict:
    """--category: "all", "clean" or one category name -> {name: cat_id}."""
    if category == "all":
        return dict(CATS_ALL)
    if category == "clean":
        return dict(clean)
    return {category: CATS_ALL[category]}


def listdir(d: str):
    return sorted(os.listdir(d))


def read_lst(test_lst_f: str):
    """Object ids of <cat_id>_test.lst, one per line, with the line ends stripped as the reference does."""
    with open(test_lst_f, "r") as f:
        return [o.rstrip("\r\n") for o in f.readlines()]


def read_mesh(engine, path):
    """OBJ -> (verts, faces) through the engine's device reader (Engine.read_obj, bit for bit create_sdf.read_obj).  An
    engine without a device reader -- a CPU stand-in for the evaluation methods -- reads with create_sdf.read_obj."""
    reader = getattr(engine, "read_obj", None)
    return reader(path) if reader is not None else read_obj(path)
