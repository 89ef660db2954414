"""Compare the SASS of two builds of the library function by function (no GPU): every kernel of the first must compile to
the same instructions in the second.  Kernels only in the second are listed as NEW.

  python scripts/sass_compare.py old/libtmd_b200.so torchmd_b200/libtmd_b200.so
"""
import re, subprocess, sys

def funcs(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    table, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1); table[cur] = []; continue
        if cur and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            ins = re.sub(r"/\*[0-9a-f]{4}\*/", "", line.split(";")[0]).strip()
            table[cur].append(ins)
    return table

a, b = funcs(sys.argv[1]), funcs(sys.argv[2])
same = diff = 0
missing = []
for name, body in a.items():
    if name not in b:
        missing.append(name); continue
    if body == b[name]: same += 1
    else:
        diff += 1; print("DIFF", name)
print(f"parent functions: {len(a)}, identical: {same}, different: {diff}, missing: {len(missing)}; new functions: {len(set(b) - set(a))}")
for n in missing: print("MISSING", n)
for n in sorted(set(b) - set(a)): print("NEW", n)
