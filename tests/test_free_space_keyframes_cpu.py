"""Host side of so_map_clear_free_space_keyframes: the keyframe cull (so_free_rule.h) never skips a (block, keyframe) pair that holds
a map point in range, on random and adversarial points (tests/cpp/free_rule_test.cpp); the entry declared, exported and bound; the
shim's new members compiling."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cull_never_skips_a_point_in_range(tmp_path):
    exe = tmp_path / "free_rule_test"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-ffp-contract=off",
                           os.path.join(ROOT, "tests", "cpp", "free_rule_test.cpp"), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    print(out.stdout.strip())
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout


def test_tile_budget_is_stated_in_the_header():
    with open(os.path.join(ROOT, "superodom_b200", "csrc", "so_free_rule.h")) as f:
        rule = f.read()
    assert re.search(r"kFreeTileBytes = size_t\(256\) << 20;", rule)
    with open(os.path.join(ROOT, "include", "superodom_b200.h")) as f:
        hdr = f.read()
    assert "256 MiB (kFreeTileBytes" in hdr
    assert re.search(r"int so_map_clear_free_space_keyframes\(so_ctx\* dst, so_ctx\* src, const int32_t\* ids, size_t n_ids, "
                     r"const double\* poses7, int stores,\s+const so_free_space\* opts, so_free_space_keyframes_result\* result\);", hdr)


def test_entry_exported_and_bound():
    from superodom_b200 import api, build
    assert "so_map_clear_free_space_keyframes" in api.EXPORTS
    lib = build.build()
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    assert re.search(r"\bso_map_clear_free_space_keyframes\b", syms)
    L = api.load_library()
    assert len(L.so_map_clear_free_space_keyframes.argtypes) == 8
    assert [n for n, _ in api.FreeSpaceKeyframesResult._fields_] == ["n_keyframes", "n_image_points", "n_pixels_hit", "n_candidates",
                                                                     "n_removed", "n_after", "n_tiles", "time_ms"]
    import ctypes as C
    assert C.sizeof(api.FreeSpaceKeyframesResult) == 9 * 8


def test_shim_members_compile(tmp_path):
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "keyframe_clear_test.cpp")])
