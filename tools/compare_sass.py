"""Per-kernel SASS comparison of two builds of libf3dgs_b200.so (no GPU needed):

    python tools/compare_sass.py OLD/libf3dgs_b200.so NEW/libf3dgs_b200.so

An opt-in feature usually adds a trailing `bool` template flag (default false) and trailing kernel parameters, which
change the mangled names of the existing instantiations.  So every kernel of OLD is matched with the kernel of NEW whose
demangled name is the same after trailing `false` template arguments are dropped and whose parameter list starts with
OLD's, and their instruction streams (addresses and encodings stripped) are compared.  Prints one line per kernel that
differs or has no counterpart, a summary, and NEW's kernels without an OLD counterpart; exits 1 if any OLD kernel differs
or is missing.  Needs cuobjdump and c++filt on PATH.
"""
import re
import subprocess
import sys


def kernels(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            if cur:
                funcs[cur] = body
            cur, body = m.group(1), []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;?\s*(/\*.*\*/)?\s*$", line)
        if cur and m:
            body.append(m.group(1))
    if cur:
        funcs[cur] = body
    names = list(funcs)
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return {re.sub(r"^void ", "", d): funcs[n] for n, d in zip(names, dem)}


def split(d):
    """demangled name -> (name with trailing `false` template arguments dropped, parameter list)"""
    i, depth = len(d), 0
    if d.endswith(")"):  # the parenthesis that opens the parameter list matches the last one
        for i in range(len(d) - 1, -1, -1):
            depth += {")": 1, "(": -1}.get(d[i], 0)
            if depth == 0:
                break
    name, params = d[:i], d[i:]
    while True:
        n = re.sub(r"(<[^<>]*?)(, false)>$", r"\1>", name)
        n = re.sub(r"<false>$", "", n)
        if n == name:
            return name, params
        name = n


def main(old_lib, new_lib):
    old, new = kernels(old_lib), kernels(new_lib)
    new_split = [(d, *split(d)) for d in new]
    matched, same, bad = set(), 0, 0
    for d, body in sorted(old.items()):
        name, params = split(d)
        cands = [nd for nd, nn, np_ in new_split if nn == name and np_.rstrip(")").startswith(params.rstrip(")"))]
        if not cands:
            print("MISSING", d)
            bad += 1
            continue
        matched.update(cands)
        if any(new[c] == body for c in cands):
            same += 1
        else:
            print("DIFFERS", d, f"({len(body)} vs {len(new[cands[0]])} instructions)")
            bad += 1
    print(f"{len(old)} kernels in {old_lib}: {same} with identical SASS in {new_lib}, {bad} differ or are missing")
    for d in sorted(set(new) - matched):
        print("NEW", d)
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
