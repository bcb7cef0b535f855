"""Compares the SASS of every kernel instance in two `cuobjdump -sass` dumps, function by function.

  python tools/sass_compare.py parent.sass new.sass

Each dump is the concatenated `cuobjdump -sass` of the cubins of one tree (nvcc -cubin -gencode arch=compute_90a,code=sm_90a with the
flags of _lib.NVCC_FLAGS, one .cu at a time).  The anonymous-namespace hashes in the mangled names (both the prefix and the one after the file name) depend on the file's
contents, so they are normalised; instructions are compared without their addresses and encodings.  Functions present in only one dump are listed
(a new kernel is expected there); every function present in both must be identical.
"""
import re, sys
def funcs(path):
    out, cur = {}, None
    for line in open(path):
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = re.sub(r'(_GLOBAL__N__X_\d+_\w+?_cu_)[0-9a-f]{8}', r'\1X', re.sub(r'_GLOBAL__N__[0-9a-f]+_', '_GLOBAL__N__X_', m.group(1))); out[cur] = []; continue
        if cur is None: continue
        m = re.match(r'\s*/\*([0-9a-f]{4,})\*/\s*(.*?);', line)
        if m: out[cur].append(m.group(2).strip())
    return out
a, b = funcs(sys.argv[1]), funcs(sys.argv[2])
ok = True
for k in sorted(set(a) | set(b)):
    if k not in a or k not in b:
        print("only in one:", k, k in a, k in b); ok = False if k in a else ok
        continue
    if a[k] == b[k]:
        print("same  %5d  %s" % (len(a[k]), k)); continue
    ok = False
    n = next((i for i, (x, y) in enumerate(zip(a[k], b[k])) if x != y), min(len(a[k]), len(b[k])))
    print("DIFF  %5d vs %5d  first at %d: %r vs %r  %s" % (len(a[k]), len(b[k]), n, a[k][n] if n < len(a[k]) else None, b[k][n] if n < len(b[k]) else None, k))
print("ALL PRE-EXISTING SAME" if ok else "DIFFERENCES")
