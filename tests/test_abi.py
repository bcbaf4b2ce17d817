"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and
exports every symbol include/plslam_b200.h declares; the product path fails loudly without a GPU."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "plslam_b200.h")).read()
    return sorted(set(re.findall(r"PLS_API\s+(?:const\s+char\*|int)\s+(pls_\w+)\s*\(", text)))


def test_library_builds_and_exports_every_declared_symbol():
    from pylidar_slam_b200 import _lib, build
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    declared = _declared()
    assert len(declared) >= 30
    assert "pls_kdmap_knn" in declared  # the test aid of the normals' neighbour lists
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert sorted(_lib.exported_symbols()) == declared, "ctypes signature table and header disagree"
    assert b"sm_90a" in _lib.load().pls_version()


def test_sass_is_sm_90a_only():
    import subprocess
    from pylidar_slam_b200 import build
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", build.build()], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from pylidar_slam_b200 import _lib
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.Context()


def test_product_path_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "pylidar_slam_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in text or f == "synthetic.py", f"{f} mentions the oracle"


def test_sass_carries_the_hopper_features_the_design_names():
    """The projective correspondence kernel really issues TMA bulk copies completed on mbarriers (UBLKCP / SYNCS), the kd
    kernels really reduce with warp-wide redux (REDUX on sm_90a); nothing pulls in a library kernel (every kernel of
    the .so is ours).  tools/sass_census.py over the built library; needs cuobjdump, no GPU."""
    import shutil
    import subprocess
    import sys
    if not (shutil.which("cuobjdump") or os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("cuobjdump not available")
    from pylidar_slam_b200 import build
    build.build()
    env = {**os.environ, "PATH": os.environ.get("PATH", "") + ":/usr/local/cuda/bin"}
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_census.py")], capture_output=True, text=True, env=env).stdout
    rows = {l.split()[0]: l for l in out.splitlines() if l and not l.startswith("#")}

    def count(kernel, op):
        m = re.search(rf"\b{op}=(\d+)", rows[kernel])
        return int(m.group(1)) if m else 0

    assert "sm_90a" in out.splitlines()[0] and len(rows) > 60
    assert count("proj_icp_tma_kernel", "UBLKCP") >= 1 and count("proj_icp_tma_kernel", "SYNCS") >= 1
    assert count("kd_nn_warp_kernel", "REDUX") >= 1 and count("kd_normals_warp_kernel", "REDUX") >= 1
    assert not any(k.startswith(("cub::", "thrust::", "cutlass", "cublas")) for k in rows)
