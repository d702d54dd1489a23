"""
Compare the SASS of every kernel in two builds of libgnm.so (`cuobjdump -sass`, instructions and encodings, addresses dropped):
prints the kernels only one build has and the common kernels whose code differs.  Exit status 1 if any common kernel differs.

    python tools/sass_diff.py OLD/libgnm.so NEW/libgnm.so
"""
import re
import shutil
import subprocess
import sys


def kernels(lib: str) -> dict:
    cob = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cob, "-sass", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for part in sass.split("Function : ")[1:]:
        name, body = part.split("\n", 1)
        lines = (re.sub(r"/\*[0-9a-f]{4,}\*/", "", ln).strip() for ln in body.split(".section")[0].splitlines())
        out[name.strip()] = "\n".join(ln for ln in lines if ln)
    return out


def main():
    a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
    print("only in the first:", sorted(set(a) - set(b)))
    print("only in the second:", sorted(set(b) - set(a)))
    diff = sorted(n for n in set(a) & set(b) if a[n] != b[n])
    print(f"{len(set(a) & set(b))} common kernels, {len(diff)} differ: {diff}")
    sys.exit(1 if diff else 0)


if __name__ == "__main__":
    main()
