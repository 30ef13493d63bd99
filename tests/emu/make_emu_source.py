"""TEST INFRASTRUCTURE: writes a g++-compilable scratch copy of featurebase_b200/csrc (the product sources stay untouched).

Three rewrites, each checked to hit at least the expected number of sites (an unknown construct fails the build loudly):
  * kernel<<<grid, block, smem, stream>>>(args);   ->  emu::launch(grid, block, smem, [&] { kernel(args); });
  * extern __shared__ T name[];                     ->  T* name = reinterpret_cast<T*>(emu::g_dyn);
  * inline PTX: the handful of statements the kernels use (tests/emu/cuda_runtime.h); any other inline PTX fails the rewrite
"""
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "featurebase_b200", "csrc")


def _match_back(s, end):
    """start index of the callee expression that ends at `end` (exclusive): identifier[<...>] or a parenthesised expression"""
    i = end
    if s[i - 1] == ")":
        depth = 0
        while True:
            i -= 1
            depth += s[i] == ")"
            depth -= s[i] == "("
            if depth == 0:
                return i
    if s[i - 1] == ">":
        depth = 0
        while True:
            i -= 1
            depth += s[i] == ">"
            depth -= s[i] == "<"
            if depth == 0:
                break
    while i > 0 and (s[i - 1].isalnum() or s[i - 1] in "_:"):
        i -= 1
    return i


def _match_fwd(s, start, open_ch, close_ch):
    depth, i = 0, start
    while True:
        depth += s[i] == open_ch
        depth -= s[i] == close_ch
        i += 1
        if depth == 0:
            return i


def rewrite_launches(s):
    n = 0
    while True:
        k = s.find("<<<")
        if k < 0:
            return s, n
        c0 = _match_back(s, k)
        e = s.find(">>>", k)
        cfg = s[k + 3:e]
        a0 = e + 3
        assert s[a0] == "(", s[a0:a0 + 40]
        a1 = _match_fwd(s, a0, "(", ")")
        parts, depth, cur = [], 0, ""
        for ch in cfg:                                   # split the launch configuration on top-level commas
            depth += ch in "(<"
            depth -= ch in ")>"
            if ch == "," and depth == 0:
                parts.append(cur)
                cur = ""
            else:
                cur += ch
        parts.append(cur)
        while len(parts) < 3:
            parts.append("0")
        callee, args = s[c0:k], s[a0:a1]
        s = s[:c0] + f"emu::launch({parts[0]}, {parts[1]}, {parts[2]}, [&] {{ {callee}{args}; }})" + s[a1:]
        n += 1


ASM = [
    (r'asm volatile\("ld\.global\.nc\.L1::no_allocate\.v4\.u32 \{%0,%1,%2,%3\}, \[%4\];" : "=r"\(r\.x\), "=r"\(r\.y\), "=r"\(r\.z\), "=r"\(r\.w\) : "l"\(p\)\);', "r = *p;"),
    (r'asm volatile\("prefetch\.global\.L2 \[%0\];" :: "l"\(p\)\);', "(void)p;"),
    (r'asm volatile\("prefetch\.global\.L2 \[%0\];" :: "l"\(np \+ \(unsigned long long\)\(lane & 15\) \* 128ull\)\);', "(void)np;"),
    (r'asm volatile\("ld\.global\.nc\.L1::no_allocate\.v2\.u32 \{%0,%1\}, \[%2\];" : "=r"\(r\.x\), "=r"\(r\.y\) : "l"\(p\)\);', "r = *p;"),
    (r'asm volatile\("bar\.sync %0, 64;" :: "r"\(id\) : "memory"\);', "emu::named_barrier(id, 64);"),
    (r'asm volatile\("red\.shared\.or\.b32 \[%0\], %1;" :: "r"\((\w+)\), "r"\(([^()]+)\) : "memory"\);', r"emu::red_or(\1, \2);"),
    (r'asm volatile\("red\.shared\.and\.b32 \[%0\], %1;" :: "r"\((\w+)\), "r"\(([^()]+)\) : "memory"\);', r"emu::red_and(\1, \2);"),
    (r'asm volatile\("red\.shared\.xor\.b32 \[%0\], %1;" :: "r"\((\w+)\), "r"\(([^()]+)\) : "memory"\);', r"emu::red_xor(\1, \2);"),
    (r'asm volatile\("" : "\+r"\(([\w\[\].]+)\)\);', r"(void)\1;"),
    (r'asm volatile\("" : "\+l"\((\w+)\)\);', r"(void)\1;"),
    (r'asm volatile\("cp\.async\.cg\.shared\.global \[%0\], \[%1\], 16;" :: "r"\(\(uint32_t\)__cvta_generic_to_shared\(dst_smem\)\), "l"\(src\) : "memory"\);', r"*dst_smem = *src;"),
    (r'asm volatile\("cp\.async\.commit_group;" ::: "memory"\);', r"(void)0;"),
    (r'asm volatile\("cp\.async\.wait_group %0;" :: "n"\(N\) : "memory"\);', r"(void)0;"),
    (r'asm volatile\("ld\.shared\.u32 %0, \[%1\];" : "=r"\((\w+)\) : "r"\((\w+)\)\);', r"\1 = emu::lds_u32(\2);"),
    (r'asm volatile\("st\.shared\.u32 \[%0\], %1;" :: "r"\((\w+)\), "r"\(([^()]+)\) : "memory"\);', r"emu::sts_u32(\1, \2);"),
]


def rewrite_asm(s):
    n = 0
    for pat, rep in ASM:
        s, k = re.subn(pat, rep, s)
        n += k
    left = re.findall(r'\basm\s*(?:volatile\s*)?\((?:[^;"]|"(?:[^"\\]|\\.)*")*\);', s)
    if left:
        raise RuntimeError("inline PTX without an emulation (add it to ASM and tests/emu/cuda_runtime.h): " + "; ".join(left))
    return s, n


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    report = {}
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".h")):
            continue
        s = open(os.path.join(CSRC, name)).read()
        s, n_launch = rewrite_launches(s)
        s, n_dyn = re.subn(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?(\w+)\s+(\w+)\[\];", r"\1* \2 = reinterpret_cast<\1*>(emu::g_dyn);", s)
        s, n_asm = rewrite_asm(s)
        s = s.replace('#include "../../include/fbgpu.h"', f'#include "{os.path.join(ROOT, "include", "fbgpu.h")}"')
        out = name[:-3] + ".cpp" if name.endswith(".cu") else name
        open(os.path.join(out_dir, out), "w").write(s)
        report[name] = (n_launch, n_dyn, n_asm)
    tot = [sum(v[i] for v in report.values()) for i in range(3)]
    assert tot[0] >= 9 and tot[1] >= 4 and tot[2] >= 8, f"rewrite counts changed, look at the sources: {report}"
    return report


if __name__ == "__main__":
    print(main(sys.argv[1]))
