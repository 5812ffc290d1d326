#!/bin/bash
# Developer script: is the device code (SASS of every kernel) of the working tree's libpb2.so the same as that of <commit>?
# Builds <commit> in a temporary worktree and compares `cuobjdump -sass` function by function: the bodies of the two
# listings as multisets, with the `Function :` lines (the names) and the translation unit's hash in anonymous-namespace
# names masked, so renamed kernels and template arguments still pair up.  Prints both function counts and every body that
# has no twin on the other side.  Used after refactors and host-only changes to pb2_cuda.cu: the kernels that were
# verified on the GPU are then provably the ones that ship.
# usage: tools/same_device_code.sh <commit>
set -e
cd "$(dirname "$0")/.."
wt=$(mktemp -d /tmp/pb2_wt.XXXXXX)
git worktree add -q "$wt" "$1"
trap 'git worktree remove --force "$wt"; git worktree prune' EXIT
make -C "$wt/pbrt_v3_b200/csrc" -j8 > "$wt/build.log" 2>&1
cuobjdump -sass "$wt/pbrt_v3_b200/lib/libpb2.so" > "$wt/a.sass"
cuobjdump -sass pbrt_v3_b200/lib/libpb2.so > "$wt/b.sass"
python3 - "$1" "$wt/a.sass" "$wt/b.sass" <<'EOF'
import collections, re, sys

def bodies(path):
    """{masked body: [function names]} of one listing"""
    out, name, body = collections.defaultdict(list), None, []
    for line in open(path):
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name, body = m.group(1), []
        elif name is not None and re.fullmatch(r"\s*\.{10}\s*", line):   # the end of a function
            out["".join(body)].append(name)
            name = None
        elif name is not None:
            body.append(re.sub(r"_GLOBAL__N__[0-9a-f]*_", "_GLOBAL__N__X_", line))
    return out

a, b = bodies(sys.argv[2]), bodies(sys.argv[3])
print(f"{sys.argv[1]}: {sum(map(len, a.values()))} functions; working tree: {sum(map(len, b.values()))} functions")
differ = False
for side, mine, other in ((sys.argv[1], a, b), ("working tree", b, a)):
    for body, names in mine.items():
        for name in names[len(other.get(body, [])):]:
            print(f"no twin, {side}: {name}")
            differ = True
print("device code DIFFERS" if differ else "device code identical")
sys.exit(1 if differ else 0)
EOF
