"""Writes tests/golden/window_without_frames.npz: window buffers of windows WITHOUT tracked frames, made by a build of the
commit before tracked frames were added (f2f8567), so that the tests can check that a window without frames still gives
that build's buffer bit for bit (WindowBlocks.pack on the host, dfk_window_assemble_geometric on the device).

    python tests/golden/make_window_f0_fixture.py <checkout of f2f8567 with its libdfk.so built> [out.npz]

Needs a GPU (the device buffer).  Per code size C in (8, 32): random Gram records of a 4-keyframe window (ring pairs,
one pair each way, a self pair, 2 levels per pair) with two sparse geometric links, the parent's pack of them and the
parent's device buffer."""
import os
import sys

import numpy as np


def inputs(cs, rng):
    K = 4
    pairs = [(k, (k + 1) % K) for k in range(K)] + [(1, 0), (2, 2)]
    item_pair = [p for p in range(len(pairs)) for _ in range(2)]
    sizes = [(40 >> l, 30 >> l) for _ in pairs for l in range(2)]
    n, NP = len(item_pair), 12 + cs
    A = rng.standard_normal((n, 2 * NP, NP + 1))
    JtJ = np.einsum("nri,nrj->nij", A[..., :NP], A[..., :NP]).astype(np.float32)
    Jtr = np.einsum("nri,nr->ni", A[..., :NP], A[..., NP]).astype(np.float32)
    res = np.einsum("nr,nr->n", A[..., NP], A[..., NP]).astype(np.float32)
    inl = rng.integers(50, 500, n)
    nh = NP * (NP + 1) // 2
    iu = np.triu_indices(NP)
    rec = np.zeros((n, nh + NP + 2), np.float32)
    rec[:, :nh] = JtJ[:, iu[0], iu[1]]
    rec[:, nh:nh + NP] = Jtr
    rec[:, nh + NP] = res
    rec[:, nh + NP + 1] = inl.astype(np.uint32).view(np.float32)
    geo_pairs = [(0, 2), (3, 1)]
    NG = 12 + 2 * cs
    G = rng.standard_normal((len(geo_pairs), 2 * NG, NG + 1))
    gJ = np.einsum("nri,nrj->nij", G[..., :NG], G[..., :NG]).astype(np.float32)
    gr = np.einsum("nri,nr->ni", G[..., :NG], G[..., NG]).astype(np.float32)
    ngh = NG * (NG + 1) // 2
    ig = np.triu_indices(NG)
    geo = np.zeros((len(geo_pairs), ngh + NG + 2), np.float32)
    geo[:, :ngh] = gJ[:, ig[0], ig[1]]
    geo[:, ngh:ngh + NG] = gr
    geo[:, ngh + NG] = 1.0
    return K, pairs, item_pair, sizes, rec, geo_pairs, geo


def main():
    parent = os.path.abspath(sys.argv[1])
    out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                             "window_without_frames.npz")
    sys.path.insert(0, parent)  # the parent's package and its libdfk.so
    import torch
    import deepfactors_b200
    from deepfactors_b200 import factors
    from deepfactors_b200.aligners import SfmAligner, Window
    assert os.path.dirname(os.path.abspath(deepfactors_b200.__file__)) == os.path.join(parent, "deepfactors_b200")
    data = {}
    for cs in (8, 32):
        K, pairs, item_pair, sizes, rec, geo_pairs, geo = inputs(cs, np.random.default_rng(1234 + cs))
        H, g, r_, n_ = factors.unpack_records(rec, cs)
        gH, gg, gres, _ = factors.unpack_geometric_records(geo, cs)
        lay = factors.WindowBlocks(K, cs, pairs, geo_pairs)
        pack = lay.pack(item_pair, H, g, r_, n_, sizes, geo=(gH, gg, gres))
        win = Window(SfmAligner(cs), K, pairs, item_pair, sizes, geo_pairs)
        dev = win.assemble(torch.from_numpy(rec).cuda(), geo_records=torch.from_numpy(geo).cuda()).cpu().numpy()
        for name, v in dict(K=K, pairs=pairs, item_pair=item_pair, sizes=sizes, records=rec, geo_pairs=geo_pairs,
                            geo_records=geo, pack=pack, device=dev).items():
            data[f"c{cs}_{name}"] = np.asarray(v)
    np.savez_compressed(out, **data)
    print(f"wrote {out}")


if __name__ == "__main__":
    main()
