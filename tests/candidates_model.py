"""What matching a view pair against caller-given candidates (Line3D::setLineCandidates, l3d_match_pairs_cand) must produce, stated on
the oracle's keep-all rows: a row keeps the members of its full survivor set whose target segment is a candidate, then the kNN rule.

    restricted(row) = topk(keep_all(row) ∩ candidates)

keep_all(row) is every target with overlap > epi and all four depths in front (pyoracle.match_lines(..., knn=0), ascending tgt_seg);
the kNN rule is the matcher's: 1 <= kNN: the kNN best by overlap descending, the smaller tgt_seg first on a tie; kNN <= 0: all of
them in ascending tgt_seg."""
import numpy as np

from line3dpp_b200 import synth
from oracle import pyoracle


def restricted_rows(keep_all_rows, candidates, knn):
    """keep_all_rows: (counts int32[Ns], matches[Ns, cap]) of pyoracle.match_lines(..., knn=0) (MATCH_DT), or any rows of that kind
    with tgt_seg and overlap fields; candidates: (src_seg, tgt_seg) pairs ([n, 2], duplicates allowed) or None for every target.
    Returns (counts int32[Ns], matches[Ns, cap']) of the same dtype, cap' = knn for knn > 0, else the input's cap."""
    counts, rows = keep_all_rows
    Ns = len(counts)
    cap = knn if knn > 0 else rows.shape[1]
    allowed = None
    if candidates is not None:
        allowed = [set() for _ in range(Ns)]
        for s, t in np.asarray(candidates, np.int64).reshape(-1, 2):
            allowed[int(s)].add(int(t))
    out_c = np.zeros(Ns, np.int32)
    out = np.zeros((Ns, cap), rows.dtype)
    for r in range(Ns):
        row = rows[r, :counts[r]]
        if allowed is not None:
            row = row[np.fromiter((int(t) in allowed[r] for t in row["tgt_seg"]), bool, len(row))]
        if knn > 0:
            row = row[np.lexsort((row["tgt_seg"], -row["overlap"].astype(np.float64)))][:knn]
        out_c[r] = len(row)
        out[r, :len(row)] = row
    return out_c, out


def pair_keep_all(scene, src, tgt, epi, f64, fn=None):
    """the oracle's keep-all rows of one view pair (view indices) with the inputs matchImages gives it: REF_GPU the float F and
    camera blocks (untranslated centres), REF_CPU the double ones.  fn: another matcher of orc_match_lines_f32's signature (the
    verbatim reference wrapper, pyoracle.ref_lib().ref_match_lines)"""
    RtKinv, C = synth.camera_blocks(scene)
    F = synth.fundamental(scene.K[src], scene.R[src], scene.t[src], scene.K[tgt], scene.R[tgt], scene.t[tgt])
    fn = fn or (pyoracle.lib().orc_match_lines_f64 if f64 else pyoracle.lib().orc_match_lines_f32)
    c, m, _, _ = pyoracle.match_lines(fn, scene.segs[src], scene.segs[tgt], F.reshape(9), RtKinv[src].reshape(9), RtKinv[tgt].reshape(9),
                                      C[src], C[tgt], int(scene.cam_ids[src]), int(scene.cam_ids[tgt]), epi, 0, f64=f64,
                                      cap=max(len(scene.segs[tgt]), 1))
    return c, m


def match_source(scene, lists, epi=0.25, fn=None):
    """an OraclePipeline(use_gpu=True, match_source=...) source that matches every view pair as setLineCandidates(lists) restricts it:
    lists {(camA, camB): [n, 2] (segment of camA, segment of camB)}, either camera order; pairs without a list are scanned; fn as for
    pair_keep_all"""
    index = {int(c): i for i, c in enumerate(scene.cam_ids)}
    norm = {}
    for (a, b), v in lists.items():
        v = np.asarray(v, np.int64).reshape(-1, 2)
        norm[(min(a, b), max(a, b))] = v if a < b else v[:, ::-1]

    def source(src_cam, tgt_cam, Ns, Nt, knn, cap):
        key = (min(src_cam, tgt_cam), max(src_cam, tgt_cam))
        cand = norm.get(key)
        if cand is not None and src_cam > tgt_cam:
            cand = cand[:, ::-1]
        c, m = restricted_rows(pair_keep_all(scene, index[src_cam], index[tgt_cam], epi, False, fn), cand, knn)
        out = np.zeros((Ns, cap), pyoracle.MATCH_DT)
        out[:, :min(cap, m.shape[1])] = m[:, :cap]
        return c, out
    return source
