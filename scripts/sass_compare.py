"""Checks that a change leaves existing kernels alone: every kernel of the OLD objects must appear among the NEW objects'
kernels with the same SASS, instruction for instruction (`cuobjdump -sass`, encodings aside, mangled names aside --
template parameters that grew a value or a trailing parameter change the name, not the code).
Usage: python scripts/sass_compare.py OLD_CSRC_DIR NEW_CSRC_DIR   (directories holding the gs_*.o of two builds)"""
import collections
import glob
import os
import re
import subprocess
import sys


def kernels(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = fns.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(.*?)\s*;?\s*(/\*.*\*/)?\s*$", line)
        if m and cur is not None:
            cur.append(re.sub(r"\b_Z\w+", "NAME", m.group(1)))
    return {k: "\n".join(v) for k, v in fns.items()}


def main(old_dir, new_dir):
    missing = checked = 0
    for old in sorted(glob.glob(os.path.join(old_dir, "*.o"))):
        new = os.path.join(new_dir, os.path.basename(old))
        o, n = kernels(old), (kernels(new) if os.path.exists(new) else {})
        have = collections.Counter(n.values())
        for name, body in o.items():
            checked += 1
            if have[body] == 0:
                missing += 1
                demangled = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
                print(f"CHANGED {os.path.basename(old)}: {demangled}")
        print(f"{os.path.basename(old)}: {len(o)} kernels before, {len(n)} after")
    print(f"{checked} kernels checked, {missing} changed")
    return 1 if missing else 0


if __name__ == "__main__":
    sys.exit(main(*sys.argv[1:3]))
