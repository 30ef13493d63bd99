#!/usr/bin/env python
"""Which kernels of the current build differ, instruction for instruction, from the build of an earlier commit?
    python tools/sass_diff.py <commit>         # e.g. the last commit whose library was parity-tested and timed on an H100
Builds that commit's csrc/ in a scratch directory with the same nvcc line, dumps both libraries with cuobjdump -sass and
compares the instruction streams per kernel (addresses and encodings stripped; template arguments that did not exist yet
or no longer exist are matched by kernel name: an untemplated kernel and its <false> instantiation, groupby_values_kernel's
<GvAgg(0)> / <GvAgg(1)> (count only / Sum) and row_count_kernel's <RcOut(0)> / <RcOut(1)> (summed / per shard) and the
<false> / <true> of the bool templates they replaced).  Kernels of the old
build that the new one lacks are reported DELETED.  No GPU needed.  A kernel reported IDENTICAL is, bit for bit in its
instructions, the one that was parity-tested and timed on the device."""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from featurebase_b200.build import ARCH  # noqa: E402


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            res[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,5}\*/\s+(.*?);", line)
        if m and cur:
            res[cur].append(m.group(1).strip())
    return res


ENUM_AS_BOOL = {"LNS_5GvAggE0": "Lb0", "LNS_5GvAggE1": "Lb1",     # GvAgg::kCount / kSum took the place of <false> / <true>
                "LNS_5RcOutE0": "Lb0", "LNS_5RcOutE1": "Lb1"}     # and row_count_kernel's RcOut::kSummed / kPerShard


def short(name):
    """(kernel name, template argument) with the argument as mangled: Lb0 / Lb1 for a bool, LNS_<n><Enum>E<value> for an enum"""
    m = re.match(r"_ZN5fbgpu\d+([a-z_0-9]+?)(I(Lb[01]|LNS_\d+\w+?E\d+)E)?E", name)
    return (m.group(1), m.group(3) or "") if m else (name, "")


def label(name, targ):
    m = re.match(r"LNS_\d+(\w+?)E(\d+)$", targ)
    return name + ("<%s(%s)>" % m.groups() if m else "<%s>" % ("true" if targ == "Lb1" else "false") if targ else "")


def same_arg(a, b):
    a, b = ENUM_AS_BOOL.get(a, a), ENUM_AS_BOOL.get(b, b)
    return a == b or {a, b} <= {"", "Lb0"}


def main():
    commit = sys.argv[1]
    tmp = tempfile.mkdtemp(prefix="sassdiff_")
    tar = subprocess.run(["git", "-C", ROOT, "archive", commit, "featurebase_b200/csrc", "include"], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", tmp], input=tar, check=True)
    old = os.path.join(tmp, "libold.so")
    subprocess.run(["nvcc", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-lineinfo", "-gencode", ARCH,
                    "-I", os.path.join(tmp, "include"), "-o", old, os.path.join(tmp, "featurebase_b200/csrc/fbgpu.cu"), "-ldl"], check=True, stdout=subprocess.DEVNULL)
    a, b = kernels(old), kernels(os.path.join(ROOT, "featurebase_b200", "libfbgpu.so"))
    by_name, matched = {}, set()
    for k, v in a.items():
        by_name.setdefault(short(k)[0], []).append((short(k)[1], v, k))
    for k, v in b.items():
        name, targ = short(k)
        cands = by_name.get(name, [])
        hit = [x for x in cands if x[0] == targ] or [x for x in cands if same_arg(x[0], targ)]
        if not hit:
            print(f"NEW        {label(name, targ):28s} {len(v):5d} instructions")
        else:
            matched.add(hit[0][2])
            print(f"{'IDENTICAL' if hit[0][1] == v else 'CHANGED  '}  {label(name, targ):28s} {len(hit[0][1]):5d} -> {len(v):5d} instructions")
    for k, v in a.items():
        if k not in matched:
            print(f"DELETED    {label(*short(k)):28s} {len(v):5d} instructions")


if __name__ == "__main__":
    main()
