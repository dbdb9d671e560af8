"""CPU-side checks of the drop-in boundary: the in-tree shared library builds for sm_90a, loads, exports every
symbol include/superodom_b200.h declares, and refuses to work (loudly) without a GPU -- there is no CPU fallback."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "superodom_b200.h")


def _declared():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(so_[a-z0-9_]+)\s*\(", src)))


def test_header_compiles_as_c_and_cpp(tmp_path):
    for comp, flag, ext in (("gcc", "-std=c99", "c"), ("g++", "-std=c++17", "cpp")):
        f = tmp_path / f"t.{ext}"
        f.write_text('#include "superodom_b200.h"\nint main(void){ so_icp_result r; (void)r; return 0; }\n')
        subprocess.check_call([comp, flag, "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(f), "-o", str(tmp_path / "t.o")])


def test_library_builds_and_exports_every_declared_symbol():
    from superodom_b200 import api, build
    lib_path = build.build()
    assert os.path.exists(lib_path)
    L = C.CDLL(lib_path)
    decl = _declared()
    assert len(decl) >= 20
    for name in decl:
        assert hasattr(L, name), f"{name} declared in the header but not exported"
    assert sorted(api.EXPORTS) == decl, "python binding and header disagree on the ABI surface"
    # SASS is sm_90a
    out = subprocess.run(["cuobjdump", "--list-elf", lib_path], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_struct_layouts_match_header(tmp_path):
    from superodom_b200 import api
    f = tmp_path / "sz.c"
    f.write_text('#include <stdio.h>\n#include "superodom_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu\\n", sizeof(so_config), sizeof(so_icp_opts), sizeof(so_icp_result), sizeof(so_corr), sizeof(so_edge_corr));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(exe)])
    a, b, c, d, e = map(int, subprocess.check_output([str(exe)]).split())
    assert (a, b, c, d, e) == (C.sizeof(api.Config), C.sizeof(api.IcpOpts), C.sizeof(api.IcpResult), api.CORR_DTYPE.itemsize,
                               api.EDGE_CORR_DTYPE.itemsize)


def test_no_cpu_fallback():
    """Without a GPU the product path must fail loudly, never compute on the CPU."""
    import torch
    from superodom_b200 import api
    if torch.cuda.is_available():
        pytest.skip("GPU present: the loud-failure path is not reachable")
    assert not api.device_available()
    with pytest.raises(api.SuperOdomError):
        api.Context()


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under superodom_b200/ or include/ may reference it."""
    for base in ("superodom_b200", "include"):
        for dp, _, fs in os.walk(os.path.join(ROOT, base)):
            for fn in fs:
                if fn.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                    txt = open(os.path.join(dp, fn), errors="ignore").read()
                    assert "so_oracle" not in txt and "from oracle" not in txt and "import oracle" not in txt, fn


def test_library_holds_only_sm_90a_images():
    """Write for H100 only: every device ELF inside the shared library is an sm_90a image (no other architecture, no PTX)."""
    import shutil
    import subprocess
    from superodom_b200 import build
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    lib = build.build()
    elfs = [ln for ln in subprocess.run([tool, "-lelf", lib], capture_output=True, text=True).stdout.splitlines() if "ELF file" in ln]
    assert elfs and all("sm_90a" in ln for ln in elfs), elfs
    ptx = [ln for ln in subprocess.run([tool, "-lptx", lib], capture_output=True, text=True).stdout.splitlines() if "PTX file" in ln]
    assert not ptx, ptx


def test_sampling_indices_match_should_process_point():
    """so_sampling_indices (host-only) == calculateSamplingRate + shouldProcessPoint (LidarSlam.cpp:346-359) restated in numpy:
    rate = max/n, keep i unless fmod(i * rate, 1) + 0.001 > rate.  This list decides which points so_register uploads first."""
    from superodom_b200 import api
    rng = np.random.default_rng(5)
    cases = [(28800, 2000), (131072, 2000), (2001, 2000), (2000, 2000), (10, 0), (50000, 4095), (1, 1), (7, 3), (240000, 2000)]
    cases += [(int(n), int(m)) for n, m in zip(rng.integers(1, 60000, 40), rng.integers(1, 4096, 40))]
    for n, mf in cases:
        got = api.sampling_indices(n, mf)
        i = np.arange(n, dtype=np.float64)
        if mf > 0 and n > mf:
            rate = np.float64(mf) / np.float64(n)
            want = np.nonzero(~(np.fmod(i * rate, 1.0) + 0.001 > rate))[0]
            assert len(want) <= mf + 1
        else:
            want = np.arange(n)
        assert np.array_equal(got, want.astype(np.uint32)), (n, mf)


def test_batch_chunking_rule(tmp_path):
    """Host logic of so_register_batch*: the chunk bounds (superodom_b200/csrc/so_chunks.h, plain C++) cover the batch in order
    in at most 16 chunks; host batches expose one 8-scan upload and then grow (8, 16, 40, 64, 128, ...) with no sliver at the end."""
    exe = tmp_path / "chunks_test"
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-O1", "-I", os.path.join(ROOT, "superodom_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "chunks_test.cpp"), "-o", str(exe)])
    out = subprocess.check_output([str(exe), "64", "256", "65"], text=True).splitlines()
    assert out == ["64: 0 8 24 64", "256: 0 8 24 64 128 256", "65: 0 8 24 65", "ok"]
