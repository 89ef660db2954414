"""Compare the SASS of two builds of the library function by function (no GPU): every kernel of the first must compile to
the same instructions in the second.  Kernels only in the second are listed as NEW.  A kernel of the first that became
the <float> instantiation of a template in the second (k_vv_first -> k_vv_first<float>, k_vv_second<true, false> ->
k_vv_second<float, true, false>) is compared with that instantiation and reported under both names.

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

def float_keys(names):
    """mangled name -> demangled name without its parameters, return type and a leading <float> template argument"""
    names = list(names)
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    keys = {}
    for n, d in zip(names, out):
        d = re.sub(r"^void ", "", d.split("(")[0])
        keys[n] = re.sub(r"<float>$", "", re.sub(r"<float, ", "<", d))
    return keys

a, b = funcs(sys.argv[1]), funcs(sys.argv[2])
missing = [n for n in a if n not in b]
new = sorted(set(b) - set(a))
renamed = {}
if missing and new:
    ka, kb = float_keys(missing), float_keys(new)
    for n in missing:
        hits = [m for m in new if kb[m] == ka[n] and kb[m] != m]
        if len(hits) == 1: renamed[n] = hits[0]
same = diff = 0
for name, body in a.items():
    other = name if name in b else renamed.get(name)
    if other is None: continue
    if body == b[other]: same += 1
    else:
        diff += 1; print("DIFF", name)
    if other != name: print("RENAMED", name, "->", other, "(identical)" if body == b[other] else "(different)")
missing = [n for n in missing if n not in renamed]
new = [n for n in new if n not in renamed.values()]
print(f"parent functions: {len(a)}, identical: {same}, different: {diff}, missing: {len(missing)}; new functions: {len(new)}")
for n in missing: print("MISSING", n)
for n in new: print("NEW", n)
