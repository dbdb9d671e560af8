"""Host side of the block archive: the world-key and window logic (superodom_b200/csrc/so_archive.h, plain C++), the PCD writer that
saves a whole map (PcdIO.hpp writePointCloud, read back bit for bit by readPointCloud), and the shim's archive members compiling."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gxx(src, exe, *extra):
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-O1", *extra, os.path.join(ROOT, "tests", "cpp", src), "-o", str(exe)])


def test_archive_keys_and_window(tmp_path):
    exe = tmp_path / "archive_test"
    _gxx("archive_test.cpp", exe, "-I", os.path.join(ROOT, "superodom_b200", "csrc"))
    assert subprocess.check_output([str(exe)], text=True).splitlines() == ["ok"]


def test_pcd_write_round_trip(tmp_path):
    """writePointCloud -> readPointCloud gives the cloud back bit for bit, NaN, infinities and negative zero included, and the
    file is the binary XYZI layout PCL writes."""
    exe = tmp_path / "pcd_write_test"
    _gxx("pcd_write_test.cpp", exe, "-I", os.path.join(ROOT, "include"))
    rng = np.random.default_rng(5)
    pts = rng.normal(0, 500, size=(5000, 4)).astype(np.float32)
    pts[3, 0], pts[7, 1], pts[11, 2], pts[13, 3], pts[17, 0] = np.nan, np.inf, -np.inf, np.nan, -0.0
    src, pcd, back = tmp_path / "in.bin", tmp_path / "map.pcd", tmp_path / "back.bin"
    src.write_bytes(pts.tobytes())
    subprocess.check_call([str(exe), str(src), str(pcd), str(back)])
    assert back.read_bytes() == pts.tobytes()
    raw = pcd.read_bytes()
    head, body = raw.split(b"DATA binary\n", 1)
    assert b"FIELDS x y z intensity\n" in head and b"TYPE F F F F\n" in head and f"POINTS {len(pts)}\n".encode() in head
    assert body == pts.tobytes()
    empty = tmp_path / "empty.bin"
    empty.write_bytes(b"")
    subprocess.check_call([str(exe), str(empty), str(tmp_path / "empty.pcd"), str(tmp_path / "empty_back.bin")])
    assert (tmp_path / "empty_back.bin").read_bytes() == b""


def test_shim_archive_members_link(tmp_path):
    """LocalMap::setArchive / archiveSize / loadPriorMap / getWholeMap and writePointCloud, used as localization mode would,
    compile and link against the in-tree library."""
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "archive_shim_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "archive_shim_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(exe)
