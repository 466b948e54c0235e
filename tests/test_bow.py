"""CPU checks of the DBoW2 retrieval's specification (include/dfk.h dfk_bow_*, DESIGN.md section 4.11):
- the loader reads the reference's small_voc (k 9, L 3, 670 nodes, 585 words of which 17 weigh 0, 48-byte
  descriptors) without OpenCV, and tolerates line wrapping;
- the C oracle (bow_oracle/) equals an independent dict-based transliteration (tests/bow_cases.py) bit for bit: the
  word of every descriptor, the vector's words and value bits, the query's ids, counts and score bits, and the score
  bits, on small_voc and on synthetic 32- and 64-byte trees, with exact ties between children, zero-weight leaves,
  repeated descriptors, empty sets, max_id -1 / 0 / middle and equal entry sums;
- two vectors with no common word score -0.0;
- LoopDetector's candidate filter, selection and DetectLocalLoop equal a transliteration of loop_detector.cpp;
- the C++ facade's BowVocabularyData::LoadText (tests/cpp/bow_test parse) reads the same arrays as the Python loader,
  from the plain and from a wrapped file;
- the ctypes layouts of the DfkBow* structs match the header."""
import ctypes
import gzip
import os
import subprocess

import numpy as np
import pytest

from bow_oracle import bow_oracle as bo
from deepfactors_b200 import aligners as A
import bow_cases as bc

ROOT = bc.ROOT


def test_loader_reads_small_voc():
    v = bc.small_voc()
    assert (v["k"], v["L"], v["weighting"], v["scoring"], v["descriptor_bytes"]) == (9, 3, 0, 0, 48)
    assert len(v["node_ids"]) == 670 and len(v["word_ids"]) == 585
    assert sorted(v["node_ids"].tolist()) == list(range(1, 671))
    assert sorted(v["word_ids"].tolist()) == list(range(585))
    at = {int(i): k for k, i in enumerate(v["node_ids"])}
    leaves = set(v["node_ids"].tolist()) - set(v["parent_ids"].tolist())
    assert leaves == set(v["word_nodes"].tolist())
    assert sum(v["weights"][at[int(n)]] == 0.0 for n in v["word_nodes"]) == 17
    assert v["weights"][at[667]] == 1.3862943611198906


def test_loader_tolerates_line_wrapping():
    with gzip.open(bc.SMALL_VOC, "rt") as f:
        text = f.read()
    a = A.parse_dbow2_vocabulary(text)
    # wrap descriptor strings in the middle, with and without an escaped line break, and break the flow mappings
    b = A.parse_dbow2_vocabulary(_wrapped(text))
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def _check_transform(voc, descs):
    orc, py = bo.Vocabulary(voc), bc.PyVocabulary(voc)
    fw, w, v = orc.transform(descs)
    pfw, pv = py.transform(descs)
    assert fw.tolist() == pfw
    pw, pvals = bc.as_arrays(pv)
    assert np.array_equal(w, pw) and np.array_equal(bc.bits(v), bc.bits(pvals))
    return fw, pv


def _check_database(entries, queries, max_results=(1, 3, 10 ** 6), max_ids=None):
    db = bo.Database()
    for e in entries:
        db.add(*bc.as_arrays(e))
    n = len(entries)
    for q in queries:
        for mr in max_results:
            for mi in (max_ids or (-1, 0, n // 2)):
                ids, sc, c = db.query(*bc.as_arrays(q), mr, mi)
                pres, pc = bc.py_query(entries, q, mr, mi)
                assert c == pc
                assert ids.tolist() == [e for e, _ in pres]
                assert np.array_equal(bc.bits(sc), bc.bits([s for _, s in pres]))
        for e in range(n):
            assert bc.bits(db.score(e, *bc.as_arrays(q))) == bc.bits(bc.py_score(entries[e], q))


def test_oracle_equals_transliteration_on_small_voc():
    voc = bc.small_voc()
    sets = [bc.near_node_descriptors(voc, s, 300) for s in range(6)]
    sets.append(np.repeat(sets[0][:20], 5, axis=0))                       # repeated descriptors
    sets.append(np.zeros((0, 48), np.uint8))                              # an empty set
    at = {int(i): k for k, i in enumerate(voc["node_ids"])}
    zero = [voc["descriptors"][at[int(n)]] for n in voc["word_nodes"] if voc["weights"][at[int(n)]] == 0.0]
    sets.append(np.array(zero, np.uint8))                                 # the zero-weight leaves themselves
    vecs, skipped = [], 0
    for d in sets:
        fw, v = _check_transform(voc, d)
        skipped += sum(w == -1 for w in fw)
        vecs.append(v)
    assert skipped > 0, "no descriptor reached a zero-weight leaf"
    _check_database(vecs[:5] + [vecs[0], vecs[7]], vecs[3:])             # entry 5 repeats entry 0: equal sums


@pytest.mark.parametrize("D", [32, 64])
def test_oracle_equals_transliteration_on_synthetic_trees(D):
    voc = bc.synthetic_voc(D, k=6, L=4, D=D)
    vecs = [_check_transform(voc, bc.near_node_descriptors(voc, 10 + s, 200, 24))[1] for s in range(8)]
    _check_database(vecs[:6] + [vecs[2]] * 3, vecs[4:])


def test_exact_ties_between_children_go_to_the_first():
    voc = bc.synthetic_voc(7, k=5, L=3, D=32, ties=True)
    orc, py = bo.Vocabulary(voc), bc.PyVocabulary(voc)
    d = bc.near_node_descriptors(voc, 3, 400, 8)
    fw, _, _ = orc.transform(d)
    assert fw.tolist() == py.transform(d)[0]
    # the second child is never chosen where it copies the first: the words of tied second children do not occur
    kids = {}
    for nid, pid in zip(voc["node_ids"], voc["parent_ids"]):
        kids.setdefault(int(pid), []).append(int(nid))
    word = {int(n): int(w) for w, n in zip(voc["word_ids"], voc["word_nodes"])}
    tied = {word[c[1]] for c in kids.values() if len(c) > 1 and c[1] in word}
    assert tied and not (tied & set(fw.tolist()))


def test_disjoint_and_empty_scores_are_negative_zero():
    s = bo.score([1, 3], [0.5, 0.5], [2, 4], [0.5, 0.5])
    assert s == 0.0 and np.signbit(s)
    assert np.signbit(bo.score([], [], [1], [1.0])) and np.signbit(bc.py_score({1: 0.5}, {2: 0.5}))
    db = bo.Database()
    db.add([1], [1.0])
    ids, sc, c = db.query([], [], 3)
    assert c == 0 and len(ids) == 0


def test_score_operand_order_matters():
    """score(a, b) and score(b, a) round differently for some pairs: the specification fixes the order"""
    rng = np.random.default_rng(0)
    differ = 0
    for _ in range(2000):
        a = {w: float(rng.random() * 10.0 ** rng.integers(-3, 1)) for w in rng.choice(50, 20, replace=False)}
        b = {w: float(rng.random() * 10.0 ** rng.integers(-3, 1)) for w in rng.choice(50, 20, replace=False)}
        ab = bo.score(*bc.as_arrays(a), *bc.as_arrays(b))
        assert bc.bits(ab)[0] == bc.bits(bc.py_score(a, b))[0]
        differ += int(bc.bits(ab)[0] != bc.bits(bc.py_score(b, a))[0])
    assert differ > 0


# ------------------------------------------------------------------------------------------- LoopDetector selection
def ref_candidates(results, curr, active_window, min_similarity):
    """loop_detector.cpp:117-139 with its types: kfid = res.Id + 1 (unsigned int), curr_kf->id size_t, active_window
    int (converted to size_t), Score double against a float"""
    out = []
    u64 = np.uint64
    for rid, score in results:
        kfid = u64(np.uint32(rid) + np.uint32(1))
        if kfid == u64(curr):
            continue
        with np.errstate(over="ignore"):
            lim = u64(curr) - u64(np.int64(active_window).astype(np.uint64))
        if kfid > lim:
            continue
        if float(score) < float(np.float32(min_similarity)):
            continue
        out.append(int(kfid))
    return out


def ref_select(cands, pwc, inl, pwk, max_dist):
    best_dist = np.float32(np.inf)
    best_id, best_pose = cands[0], None
    for i, c in enumerate(cands):
        t = np.asarray(pwc[i], np.float32)[4:] - np.asarray(pwk[i], np.float32)[4:]
        dist = np.float32(np.sqrt(np.float32(np.float32(t[0] * t[0] + t[1] * t[1]) + t[2] * t[2])))
        if np.float32(inl[i]) < np.float32(0.5):
            continue
        if dist < best_dist:
            best_dist, best_id, best_pose = dist, c, pwc[i]
    if best_dist < np.float32(max_dist):
        return True, best_id, best_pose
    return False, 1, None


def ref_local(kps, pose_cam, curr, active_window, max_dist):
    best_dist, best_id = np.float32(np.inf), kps[-1][0]
    i = len(kps) - 1
    for _ in range(active_window):
        if i < 0:
            break
        kid, pwk = kps[i]
        t = np.asarray(pose_cam, np.float32)[4:] - np.asarray(pwk, np.float32)[4:]
        dist = np.float32(np.sqrt(np.float32(np.float32(t[0] * t[0] + t[1] * t[1]) + t[2] * t[2])))
        if dist < best_dist and kid != curr:
            best_dist, best_id = dist, kid
        i -= 1
    return best_id if best_id != curr and best_dist < np.float32(max_dist) else 0


def test_loop_selection_equals_loop_detector_cpp():
    rng = np.random.default_rng(5)
    pose = lambda: np.concatenate([[0, 0, 0, 1], rng.normal(0, 0.3, 3)]).astype(np.float32)
    wrapped = 0
    for trial in range(400):
        curr = int(rng.integers(1, 30))
        aw = int(rng.integers(0, 12))
        results = [(int(e), float(s)) for e, s in zip(rng.permutation(40)[:int(rng.integers(0, 12))],
                                                      np.sort(rng.random(12))[::-1])]
        ms = float(rng.choice([0.0, 0.2, 0.35, 0.5]))
        got = A.loop_candidates(results, curr, aw, ms)
        assert got == ref_candidates(results, curr, aw, ms), (results, curr, aw)
        wrapped += curr < aw and len(got) > 0
        if got:
            pwc = [pose() for _ in got]
            pwk = [p + np.float32(rng.choice([0.0, 0.01, 0.3])) * np.array([0, 0, 0, 0, 1, 1, 1], np.float32)
                   for p in pwc]
            inl = rng.choice([0.2, 0.5, 0.8], len(got))
            md = float(rng.choice([0.05, 0.1, 0.5]))
            li = A.loop_select(got, pwc, inl, pwk, md)
            det, bid, bpose = ref_select(got, pwc, inl, pwk, md)
            assert (li.detected, li.loop_id) == (det, bid)
            if det:
                assert np.array_equal(li.pose_wc, bpose)
        kps = [(k, pose()) for k in range(1, int(rng.integers(2, 15)))]
        pc = kps[int(rng.integers(0, len(kps)))][1] + np.float32(0.02)
        assert A.detect_local_loop(kps, pc, curr, aw, 0.1) == ref_local(kps, pc, curr, aw, 0.1)
    assert wrapped > 0, "no case exercised the size_t wrap of curr - active_window"


def test_struct_layouts_match_the_header(tmp_path):
    """offsets and sizes of the DfkBow* structs as the C compiler lays them out"""
    from deepfactors_b200 import _lib
    structs = [_lib.DfkBowVocabularyDesc, _lib.DfkBowVector, _lib.DfkBowQuery, _lib.DfkBowScoreItem]
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "dfk.h"', "int main(void) {"]
    for s in structs:
        n = s.__name__
        lines.append(f'printf("{n}.size %zu\\n", sizeof({n}));')
        lines += [f'printf("{n}.{f} %zu\\n", offsetof({n}, {f}));' for f, _ in s._fields_]
    lines += ['printf("DFK_BOW_MAX_DEPTH %d\\n", DFK_BOW_MAX_DEPTH);',
              'printf("DFK_BOW_MAX_NODES %d\\n", DFK_BOW_MAX_NODES);', "return 0; }"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                         check=True).stdout.splitlines())
    for s in structs:
        n = s.__name__
        assert int(got[f"{n}.size"]) == ctypes.sizeof(s), n
        for f, _ in s._fields_:
            assert int(got[f"{n}.{f}"]) == getattr(s, f).offset, (n, f)
    assert int(got["DFK_BOW_MAX_DEPTH"]) == _lib.BOW_MAX_DEPTH
    assert int(got["DFK_BOW_MAX_NODES"]) == _lib.BOW_MAX_NODES


def _wrapped(text: str) -> str:
    wrapped = text.replace('" }', '"\n      }').replace("descriptor:\"255 ", "descriptor:\"255\n          ", 40)
    return wrapped.replace(" 0 197 ", " 0 19\\\n   7 ", 25)


@pytest.mark.parametrize("wrap", [False, True])
def test_cpp_load_text_equals_python_loader(tmp_path, wrap):
    """df::BowVocabularyData::LoadText against load_dbow2_vocabulary, array by array (the weights bit for bit)"""
    exe = os.path.join(ROOT, "tests", "cpp", "bow_test")
    with gzip.open(bc.SMALL_VOC, "rt") as f:
        text = f.read()
    if wrap:
        text = _wrapped(text)
    src, out = tmp_path / "voc.yml", tmp_path / "voc.bin"
    src.write_text(text)
    r = subprocess.run([exe, "parse", str(src), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "bow_test parse OK" in r.stdout, r.stdout + r.stderr
    want = A.parse_dbow2_vocabulary(text)
    raw = out.read_bytes()
    head = np.frombuffer(raw[:28], np.int32)
    assert head.tolist() == [want["k"], want["L"], want["weighting"], want["scoring"], want["descriptor_bytes"],
                             len(want["node_ids"]), len(want["word_ids"])]
    N, W, D = int(head[5]), int(head[6]), int(head[4])
    o = 28
    for key, dt, n in (("node_ids", np.int32, N), ("parent_ids", np.int32, N), ("weights", np.float64, N),
                       ("descriptors", np.uint8, N * D), ("word_ids", np.int32, W), ("word_nodes", np.int32, W)):
        got = np.frombuffer(raw[o:o + n * np.dtype(dt).itemsize], dt)
        o += n * np.dtype(dt).itemsize
        assert np.array_equal(got.view(np.uint8), np.ascontiguousarray(want[key], dt).reshape(-1).view(np.uint8)), key
    assert o == len(raw)
