"""Line3D on a device list without a GPU: the constructor fails loudly (no CPU fallback), and the C++ frontend that takes a device list
builds warning-free against the public headers."""
import os
import subprocess

import pytest

from line3dpp_b200 import capi, line3d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def test_device_list_without_gpu_raises():
    if _has_gpu():
        pytest.skip("a GPU is present (tests/test_multidevice_gpu.py covers unusable devices)")
    with pytest.raises(capi.L3DError, match="no usable CUDA device"):
        line3d.Line3D(neighbors_by_worldpoints=False, devices=[0, 1])


def test_empty_device_list_is_refused():
    with pytest.raises(ValueError):
        line3d.Line3D(neighbors_by_worldpoints=False, devices=[])


def test_vsfm_frontend_takes_a_device_list(tmp_path):
    from line3dpp_b200 import build
    so = build.build()
    exe = tmp_path / "vsfm_frontend"
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "examples", "vsfm_frontend.cpp"), "-I" + os.path.join(ROOT, "include"),
           "-L" + os.path.dirname(so), "-ll3d_b200", "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    nvm = tmp_path / "m.nvm"
    nvm.write_text("NVM_V3\n\n1\nimg0.jpg 1000 1 0 0 0 0 0 0 0 0\n\n1\n0 0 5 255 255 255 1 0 0 1.0 2.0\n")
    args = [str(exe), str(nvm), str(tmp_path), str(tmp_path), "0", "-1", "0"]
    for bad in ("0,x", "", "0,,1", "-1"):
        r = subprocess.run(args + [bad], capture_output=True, text=True)
        assert r.returncode == 2 and "bad device list" in r.stderr, (bad, r.returncode, r.stderr)
    r = subprocess.run(args + ["0,0"], capture_output=True, text=True)
    if _has_gpu():
        assert r.returncode == 1 and "fewer than three usable images" in r.stderr, (r.returncode, r.stderr)
    else:
        assert r.returncode == 3 and "no usable CUDA device" in r.stderr, (r.returncode, r.stderr)
