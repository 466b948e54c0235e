"""Writes tests/golden/bow_orb.npz: two more places for the DBoW2 retrieval tests and a small ORB vocabulary.

    python tests/golden/make_bow_fixture.py [out.npz]

Needs OpenCV (cv2) on the host to decode the reference's test images; the tests only read the .npz.

The four gray images are two places seen twice each: the reference's testimg/0.jpg and 25.jpg (stored here, 320 x 240,
cv2.IMREAD_GRAYSCALE) and 1047 / 1052 (already in testimg.npz).  Keys gray_0, gray_25.

The vocabulary (k = 8, L = 3, 32-byte ORB descriptors, TF_IDF, L1) is trained by a test-only, deterministic
hierarchical k-medians on the CPU ORB oracle's features (orb_oracle.detect, 500 features) of those four images plus
the tests/orb_images.py set:
- a node's descriptors are split into k clusters: the initial centres are the rows at positions j * n / k of the
  node's descriptors (in their order), then 10 rounds of assignment (Hamming distance, ties to the first centre) and
  DBoW2's majority-bit mean (a bit is set when more than half of the cluster has it); a cluster that empties keeps its
  centre;
- a node with at most k descriptors gets one child per descriptor, as DBoW2's HKmeansStep does;
- nodes are listed breadth first (ids 1, 2, ... in that order), the leaves are the words in that order;
- a word's weight is DBoW2's TF_IDF idf, log(N / N_i) over the N training images, N_i the images with the word; a word
  no image has weighs 0.
Keys voc_k, voc_L, voc_node_ids, voc_parent_ids, voc_weights, voc_descriptors [N, 32], voc_word_ids, voc_word_nodes."""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("DF_REF", "/root/reference/data/testimg")
K, LEVELS, ROUNDS = 8, 3, 10


def hamming(a: np.ndarray, c: np.ndarray) -> np.ndarray:
    """[n, m] Hamming distances of rows a [n, 32] to rows c [m, 32]"""
    x = np.bitwise_xor(a[:, None, :], c[None, :, :])
    return np.unpackbits(x, axis=2).sum(axis=2)


def majority(rows: np.ndarray) -> np.ndarray:
    bits = np.unpackbits(rows, axis=1).astype(np.int64)
    return np.packbits((2 * bits.sum(axis=0) > len(rows)).astype(np.uint8))


def split(d: np.ndarray):
    """k clusters of d: (centres, assignment)"""
    n = len(d)
    c = d[[j * n // K for j in range(K)]].copy()
    a = np.zeros(n, np.int64)
    for _ in range(ROUNDS):
        a = np.argmin(hamming(d, c), axis=1)  # argmin takes the first of equal distances
        for j in range(K):
            if (a == j).any():
                c[j] = majority(d[a == j])
    return c, a


def train(descs: np.ndarray):
    # breadth first: (parent id, descriptor rows, depth)
    node_ids, parents, cents = [], [], []
    queue = [(0, descs, 0)]
    leaves = []
    while queue:
        pid, d, depth = queue.pop(0)
        if len(d) <= K:
            groups = [(d[i], d[i:i + 1]) for i in range(len(d))]
        else:
            c, a = split(d)
            groups = [(c[j], d[a == j]) for j in range(K)]
        for cen, rows in groups:
            nid = len(node_ids) + 1
            node_ids.append(nid)
            parents.append(pid)
            cents.append(cen)
            if depth + 1 < LEVELS and len(rows) > 1:
                queue.append((nid, rows, depth + 1))
            else:
                leaves.append(nid)
    # a node that was queued but split into nothing cannot occur: every queued node has > 1 row
    has_child = set(parents)
    leaves = [n for n in node_ids if n not in has_child]
    return (np.array(node_ids, np.int32), np.array(parents, np.int32), np.array(cents, np.uint8),
            np.array(leaves, np.int32))


def main(out):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from orb_oracle import orb_oracle as oo
    from orb_images import images
    g0 = cv2.imread(os.path.join(REF, "0.jpg"), cv2.IMREAD_GRAYSCALE)
    g25 = cv2.imread(os.path.join(REF, "25.jpg"), cv2.IMREAD_GRAYSCALE)
    z = np.load(os.path.join(HERE, "testimg.npz"))
    train_imgs = [g0, g25, z["gray_1047"], z["gray_1052"]] + [v for _, v in sorted(images().items())]
    feats = [oo.detect(im, 500).descriptors for im in train_imgs]
    ids, parents, cents, leaves = train(np.concatenate(feats))
    # the tree as the vocabulary: descend each training image's features to count N_i per word
    from deepfactors_b200.aligners import parse_dbow2_vocabulary  # noqa: F401 (the loader's key names)
    from bow_oracle import bow_oracle as bo
    voc = dict(k=K, L=LEVELS, weighting=0, scoring=0, descriptor_bytes=32, node_ids=ids, parent_ids=parents,
               weights=np.zeros(len(ids)), descriptors=cents, word_ids=np.arange(len(leaves), dtype=np.int32),
               word_nodes=leaves)
    leaf_pos = {int(n): i for i, n in enumerate(ids)}
    voc["weights"][[leaf_pos[int(n)] for n in leaves]] = 1.0  # every word counts while N_i is gathered
    ov = bo.Vocabulary(voc)
    ni = np.zeros(len(leaves), np.int64)
    for f in feats:
        fw = ov.transform(f)[0]
        ni[np.unique(fw[fw >= 0])] += 1
    w = np.zeros(len(ids))
    for word, n in enumerate(leaves):
        if ni[word] > 0:
            w[leaf_pos[int(n)]] = np.log(len(feats) / ni[word])
    np.savez_compressed(out, gray_0=g0, gray_25=g25, voc_k=K, voc_L=LEVELS, voc_node_ids=ids, voc_parent_ids=parents,
                        voc_weights=w, voc_descriptors=cents, voc_word_ids=voc["word_ids"], voc_word_nodes=leaves)
    print(f"{out}: {len(ids)} nodes, {len(leaves)} words, {int((w[[leaf_pos[int(n)] for n in leaves]] == 0).sum())}"
          f" of weight 0, from {sum(len(f) for f in feats)} descriptors of {len(feats)} images")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "bow_orb.npz"))
