"""Compare the SASS of every kernel of a git revision with the working tree's, function by function.

  python scripts/sass_compare.py [REV]          (REV defaults to HEAD~1)

Both trees are compiled to cubins with the library's flags (superodom_b200/build.py) into a temporary directory; every function
of REV must be present in the working tree with identical `cuobjdump -sass` text.  Anonymous-namespace names carry a hash of the
source path, which is removed before the names are matched.  Functions only the working tree has are listed.  Exit code 1 on any
difference.  Needs nvcc and cuobjdump, no GPU."""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from superodom_b200.build import NVCC_FLAGS, SOURCES  # noqa: E402

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def cubins(tree, out):
    procs = []
    for src in SOURCES:
        if not os.path.exists(os.path.join(tree, "superodom_b200", "csrc", src)):      # a source REV does not have yet
            continue
        cmd = [os.path.join(CUDA, "bin", "nvcc"), *[f for f in NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC")], "-cubin",
               os.path.join(tree, "superodom_b200", "csrc", src), "-o", os.path.join(out, src.replace(".cu", ".cubin"))]
        procs.append(subprocess.Popen(cmd))
    if any(p.wait() for p in procs):
        raise SystemExit(f"nvcc failed in {tree}")


def functions(path):
    text = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", path], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", m.group(1))
            res[cur] = []
        elif cur is not None:
            res[cur].append(line)
    return res


def main():
    rev = sys.argv[1] if len(sys.argv) > 1 else "HEAD~1"
    with tempfile.TemporaryDirectory() as tmp:
        old_tree, old_out, new_out = (os.path.join(tmp, d) for d in ("tree", "old", "new"))
        for d in (old_tree, old_out, new_out):
            os.makedirs(d)
        archive = subprocess.run(["git", "-C", ROOT, "archive", rev], capture_output=True, check=True).stdout
        subprocess.run(["tar", "-x", "-C", old_tree], input=archive, check=True)
        cubins(old_tree, old_out)
        cubins(ROOT, new_out)
        bad = 0
        for src in SOURCES:
            name = src.replace(".cu", ".cubin")
            if not os.path.exists(os.path.join(old_out, name)):
                print(f"{src}: new source, functions {sorted(functions(os.path.join(new_out, name)))}")
                continue
            old, new = functions(os.path.join(old_out, name)), functions(os.path.join(new_out, name))
            for f, body in old.items():
                if new.get(f) != body:
                    print(f"{src}: {'missing' if f not in new else 'differs'}: {f}")
                    bad += 1
            added = [f for f in new if f not in old]
            print(f"{src}: {len(old)} functions of {rev} compared" + (f"; new: {' '.join(added)}" if added else ""))
    print("identical" if not bad else f"{bad} functions differ")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
