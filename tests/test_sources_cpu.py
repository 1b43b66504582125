"""CPU: the letter-box and crop kernels compile for sm_90a for exactly the two pixel sources (u8 BGR rows and YUV 4:2:0 frames),
without spills."""
import os
import re
import subprocess

import pytest


def _ptxas(src, tmp_path):
    from retinaface_b200.build import ARCH, COMMON, CSRC, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # one (mangled entry name, info lines) pair per kernel
    return re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\n(.*?)(?=ptxas info    : Compiling|\Z)", r.stderr, re.S)


@pytest.mark.parametrize("src,kernels", [("preprocess.cu", ("k_letterbox_batch", "k_letterbox_transposed")), ("align.cu", ("k_align_faces",))])
def test_source_kernels_compile_without_spills(src, kernels, tmp_path):
    entries = _ptxas(src, tmp_path)
    for k in kernels:
        mine = [(name, info) for name, info in entries if k in name]
        assert mine, (k, entries)
        for name, info in mine:
            assert "0 bytes spill stores, 0 bytes spill loads" in info and "0 bytes stack frame" in info, (name, info)
    names = [name for name, _ in entries]
    if src == "preprocess.cu":
        # one instantiation per kernel and source: BgrRows and YuvPlanes, nothing else
        for k in kernels:
            srcs = sorted(re.search(k + r"INS_(\d+)(\w+?)EEEv", n).group(2) for n in names if k in n)
            assert srcs == ["BgrRows", "YuvPlanes"], (k, srcs)
    else:
        assert sum("k_align_faces" in n for n in names) == 4, names      # {BgrRows, YuvPlanes} x {upright, oriented}
        assert all("BgrRows" in n or "YuvPlanes" in n for n in names if "k_align_faces" in n), names
