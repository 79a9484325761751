"""Builds the golden files of tests/test_sweep_paths_gpu.py from the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile from
the reference sources):

  * ref_gpu_wide_v1.npz: the whole verbatim pipeline on its CUDA path (libl3dref_full_gpu.so, RefFullPipeline(False, True, "gpu"))
    on the scenes W1-W3, as tests/test_ref_full_gpu.py:full_record (lists as SHA-256, a 500-row estimate sample, NSAMPLE affinity
    weights); needs a GPU;
  * ref_full_wide_cpu_v1.npz: the whole verbatim pipeline on its CPU path (libl3dref_full_cpu.so) on the scene W4, in the shape of
    make_ref_cpu_golden.py: scored and kept lists as count + SHA-256 of ids and geometry + score sum, estimates and affinity
    edges as SHA-256 + a fixed sample of ROWS values, the reconstruction in full.

    python tests/golden/make_ref_wide_golden.py [--gpu] [--cpu] [--out DIR]     # default: both, into tests/golden
"""
import argparse
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import pyoracle as po  # noqa: E402
from tests import test_sweep_paths_gpu as tw, util  # noqa: E402
from tests.golden.make_ref_cpu_golden import IDS_GEO, digest  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROWS = 500                # W4: estimates and affinity weights stored as a fixed sample of this many rows


def gpu_cases(out_dir):
    from tests import test_ref_full_gpu as tf
    out = {}
    for name in ("w1", "w2", "w3"):
        _, _, _, knn, diffusion = tw.WIDE[name]
        sc = tw.wide_scene(name)
        with tempfile.TemporaryDirectory() as tmp:
            R = po.RefFullPipeline(False, True, "gpu", folder=tmp)
            R.add_scene(sc)
            assert R.match_images(knn=knn) == 0
            assert R.reconstruct(3, diffusion) == 0
            out.update(tf.full_record(R, sc.cam_ids, [len(s) for s in sc.segs], -1.0, name + "_", tw.NSAMPLE))
            del R
        print(name, "done", flush=True)
    path = os.path.join(out_dir, os.path.basename(tw.GPU_GOLDEN))
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


def cpu_cases(out_dir):
    _, _, _, knn, _ = tw.WIDE["w4"]
    sc = tw.wide_scene("w4")
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        R = po.RefFullPipeline(False, False, "cpu", folder=tmp)
        R.add_scene(sc)
        assert R.match_images(knn=knn) == 0
        assert R.reconstruct(3, False) == 0
        out["pairs"] = R.pairs()
        for cam in sc.cam_ids:
            m = R.scored(cam)
            out[f"scored_n_{cam}"] = np.array([len(m)], np.int64)
            out[f"scored_sha_{cam}"] = digest(m, IDS_GEO)
            out[f"scored_sum_{cam}"] = np.array([m["score3D"].astype(np.float64).sum()])
            k = R.matches(cam)
            out[f"kept_n_{cam}"] = np.array([len(k)], np.int64)
            out[f"kept_sha_{cam}"] = digest(k, IDS_GEO)
            out[f"kept_sum_{cam}"] = np.array([k["score3D"].astype(np.float64).sum()])
            out[f"view_info_{cam}"] = np.array(R.view_info(cam), np.float32)
        best, P = R.estimates()
        out["est_n"], out["est_sha"], out["est_P_sample"] = np.array([len(best)]), digest(best, IDS_GEO), P[util.sample_idx(len(best), ROWS)]
        ei, ej, ew = R.affinity_raw()
        out["aff_n"], out["aff_ij"], out["aff_w_sample"] = np.array([len(ei)]), util.sha(ei, ej), ew[util.sample_idx(len(ew), ROWS)]
        out["l2g"] = R.local2global()
        out["num_lines"] = np.array([R.num_lines()], np.int64)
        out["residuals"] = R.residuals()
        out["segments3d"] = R.segments3d()
        del R
    path = os.path.join(out_dir, os.path.basename(tw.CPU_GOLDEN))
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", action="store_true")
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--out", default=HERE)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    if a.cpu or not a.gpu:
        cpu_cases(a.out)
    if a.gpu or not a.cpu:
        gpu_cases(a.out)
