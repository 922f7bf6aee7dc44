"""Compare the SASS of every kernel of two builds of libertgpu.so: each function of the first (the parent's build) must
compile to the same instructions in the second.  Addresses in the listings' comments are dropped; a function missing
from the second build counts as a difference.  Prints one line per differing function and a summary; exits 1 on any.
Usage: python tools/sass_identity.py PARENT/libertgpu.so NEW/libertgpu.so"""
import re
import subprocess
import sys


def functions(lib: str) -> dict:
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
        elif cur is not None:
            cur.append(re.sub(r"/\*[0-9a-f]{4}\*/", "", line))
    return funcs


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    bad = [name for name in old if old[name] != new.get(name)]
    for name in bad:
        print("differs" if name in new else "missing", name)
    print(f"{len(old)} functions in {sys.argv[1]}: {len(old) - len(bad)} identical; {len(new) - len(old)} new in {sys.argv[2]}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
