"""CPU checks of the DBoW2 vocabulary training (include/dfk.h, the DBoW2 training block): the sequential C oracle
against an independent Python transliteration, bit for bit; DBoW2's layout on the reference's small_voc and on every
trained vocabulary; DBoW2's save writer; the ctypes layouts of the new structs."""
import os
import subprocess

import numpy as np
import pytest

import bow_cases as bc
import bow_train_cases as bt
from bow_oracle import bow_oracle as bo
from deepfactors_b200 import _lib
from deepfactors_b200 import aligners as A


def _same(a: dict, b: dict):
    for key in ("k", "L", "weighting", "scoring", "descriptor_bytes"):
        assert int(a[key]) == int(b[key]), key
    for key in ("node_ids", "parent_ids", "descriptors", "word_ids", "word_nodes"):
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    assert np.array_equal(bc.bits(a["weights"]), bc.bits(b["weights"])), "weights"


def test_small_voc_has_dbow2s_layout():
    bt.check_dbow2_layout(bc.small_voc())


@pytest.mark.parametrize("case", bt.CASES, ids=[bt.case_id(c) for c in bt.CASES])
def test_oracle_equals_the_transliteration(case):
    x, off, k, L, seed = bt.case_data(case)
    voc, stats = bo.train(x, off, k, L, seed)
    pv, ps = bt.py_train(x, off, k, L, seed)
    _same(voc, pv)
    assert stats == ps
    assert stats["capped_nodes"] == 0
    bt.check_dbow2_layout(voc)


def test_case_list_covers_emptied_clusters_and_early_stops():
    stats = {bt.case_id(c): bo.train(*bt.case_data(c))[1] for c in bt.CASES}
    assert any(s["empty_clusters"] > 0 for s in stats.values())
    # "few" sets have fewer distinct descriptors than k: the root gets fewer than k children
    x, off, k, L, seed = bt.case_data(next(c for c in bt.CASES if c[0] == "few"))
    voc, _ = bo.train(x, off, k, L, seed)
    assert int((np.asarray(voc["parent_ids"]) == 0).sum()) < k


@pytest.mark.parametrize("name", ["v.yml", "v.yml.gz"])
def test_writer_round_trips_bit_for_bit(tmp_path, name):
    voc, _ = bo.train(*bt.case_data(bt.CASES[9]))
    path = os.path.join(tmp_path, name)
    A.save_dbow2_vocabulary(path, voc)
    _same(A.load_dbow2_vocabulary(path), voc)


def test_small_voc_parse_save_parse():
    v = bc.small_voc()
    _same(A.parse_dbow2_vocabulary(A.format_dbow2_vocabulary(v)), v)


def test_writer_matches_small_voc_text():
    """the writer reproduces DBoW2's own file line for line"""
    import gzip
    with gzip.open(bc.SMALL_VOC, "rt", encoding="ascii") as f:
        text = f.read()
    assert A.format_dbow2_vocabulary(bc.small_voc()) == text


def test_opencv_reads_a_written_file(tmp_path):
    cv2 = pytest.importorskip("cv2")
    voc, _ = bo.train(*bt.case_data(bt.CASES[8]))
    path = os.path.join(tmp_path, "v.yml.gz")
    A.save_dbow2_vocabulary(path, voc)
    fs = cv2.FileStorage(path, cv2.FILE_STORAGE_READ)
    node = fs.getNode("vocabulary")
    assert int(node.getNode("k").real()) == voc["k"] and int(node.getNode("L").real()) == voc["L"]
    nodes, words = node.getNode("nodes"), node.getNode("words")
    assert nodes.size() == len(voc["node_ids"]) and words.size() == len(voc["word_ids"])
    for i in (0, nodes.size() // 2, nodes.size() - 1):
        n = nodes.at(i)
        assert int(n.getNode("nodeId").real()) == voc["node_ids"][i]
        assert int(n.getNode("parentId").real()) == voc["parent_ids"][i]
        assert n.getNode("weight").real() == voc["weights"][i]
        assert n.getNode("descriptor").string().split() == [str(b) for b in voc["descriptors"][i]]
    fs.release()


def test_new_structs_match_the_header(tmp_path):
    src = os.path.join(tmp_path, "layout.c")
    fields = {"DfkBowTrainDesc": _lib.DfkBowTrainDesc, "DfkBowTrainStats": _lib.DfkBowTrainStats,
              "DfkBowVocabularyShape": _lib.DfkBowVocabularyShape}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "dfk.h"', "int main(void) {"]
    for name, cls in fields.items():
        lines.append(f'printf("%zu\\n", sizeof({name}));')
        for f, _ in cls._fields_:
            lines.append(f'printf("%zu\\n", offsetof({name}, {f}));')
    lines.append("return 0; }")
    open(src, "w").write("\n".join(lines))
    exe = os.path.join(tmp_path, "layout")
    subprocess.run(["gcc", "-I", os.path.join(bc.ROOT, "include"), src, "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    want = []
    for cls in fields.values():
        want.append(C_sizeof(cls))
        want += [getattr(cls, f).offset for f, _ in cls._fields_]
    assert got == want


def C_sizeof(cls):
    import ctypes
    return ctypes.sizeof(cls)


@pytest.mark.parametrize("which", ["trained", "small_voc"])
def test_facade_load_text_reads_the_writer_and_save_text_matches_it(tmp_path, which):
    """df::BowVocabularyData::LoadText reads a file save_dbow2_vocabulary wrote, and SaveText writes it back byte for
    byte (tests/cpp/bow_train_test text)"""
    voc = bo.train(*bt.case_data(bt.CASES[9]))[0] if which == "trained" else bc.small_voc()
    src, out = os.path.join(tmp_path, "in.yml"), os.path.join(tmp_path, "out.yml")
    A.save_dbow2_vocabulary(src, voc)
    exe = os.path.join(bc.ROOT, "tests", "cpp", "bow_train_test")
    r = subprocess.run([exe, "text", src, out], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "bow_train_test text OK" in r.stdout, r.stdout + r.stderr
    assert open(out).read() == open(src).read()
    _same(A.load_dbow2_vocabulary(out), voc)
