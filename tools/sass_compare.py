#!/usr/bin/env python
"""Compare the SASS of every kernel in two builds of the library, symbol by symbol under the full mangled name (addresses
and encodings stripped), and list the kernels present in only one of them.  Usage: python tools/sass_compare.py OLD.so NEW.so
Exits non-zero if any kernel differs or is missing on one side."""
import re
import subprocess
import sys


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    res, name, lines = {}, None, []
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            if name:
                res[name] = lines
            name, lines = m.group(1), []
        elif re.match(r"\s*/\*[0-9a-f]{4,}\*/", ln):  # instruction lines (offsets grow past 4 hex digits)
            lines.append(re.sub(r"/\* 0x[0-9a-f]+ \*/", "", re.sub(r"^\s*/\*[0-9a-f]{4,}\*/", "", ln)).strip())
    if name:
        res[name] = lines
    return res


old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
same = 0
for k in sorted(set(old) | set(new)):
    if k not in new:
        print("only in OLD  %6d instructions  %s" % (len(old[k]), k))
    elif k not in old:
        print("only in NEW  %6d instructions  %s" % (len(new[k]), k))
    elif old[k] != new[k]:
        print("DIFFERS      %6d -> %d instructions  %s" % (len(old[k]), len(new[k]), k))
    else:
        same += 1
print("%d kernels identical, %d in OLD, %d in NEW" % (same, len(old), len(new)))
sys.exit(0 if same == len(old) == len(new) else 1)
