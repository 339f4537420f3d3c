#!/usr/bin/env python
"""SHA-1 fingerprint of every kernel's SASS in one or two builds of libfcma_b200.so.

``cuobjdump -sass`` per kernel, the address comments dropped (they move when code elsewhere in the file changes),
hashed with SHA-1.  With two libraries the kernels whose name contains one of the filters are listed side by side, and
the kernels present in both under the same name are counted as unchanged or changed.  A kernel that became a template
has a new mangled name; its instantiation is listed next to the old name for comparison.

    python tools/sass_fingerprint.py OLD.so NEW.so svm_cv
"""
import hashlib
import re
import subprocess
import sys
from collections import defaultdict


def fingerprints(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs = defaultdict(list)
    cur = None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur is not None:
            funcs[cur].append(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).strip())
    return {k: hashlib.sha1("\n".join(v).encode()).hexdigest() for k, v in funcs.items()}


def main():
    libs = [a for a in sys.argv[1:] if a.endswith(".so")]
    filters = [a for a in sys.argv[1:] if not a.endswith(".so")]
    fps = [fingerprints(lib) for lib in libs]
    for lib, fp in zip(libs, fps):
        for name in sorted(fp):
            if not filters or any(f in name for f in filters):
                print("%s  %s  %s" % (fp[name], lib, name))
    if len(fps) == 2:
        a, b = fps
        common = [k for k in a if k in b]
        print("kernels in both builds: %d, unchanged: %d, changed: %s"
              % (len(common), sum(a[k] == b[k] for k in common), [k for k in common if a[k] != b[k]]))


if __name__ == "__main__":
    main()
