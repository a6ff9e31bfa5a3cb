"""Checks that kernels keep their SASS across a change: compiles the given csrc files of two trees with the project's nvcc flags and
compares every kernel of the old object with its namesake in the new one, instruction by instruction (addresses and encodings
stripped).  Needs nvcc and cuobjdump, no GPU.

    python scripts/sass_unchanged.py OLD_TREE NEW_TREE tgemm.cu heads_fused.cu heads.cu

A kernel whose mangled name gained trailing parameters (a kernel argument appended) is matched by prefix, and a kernel that became
a template on a bool is matched with its <false> instantiation.  Prints per file the
kernels that compile to the same SASS, those that differ and those that are new; exits 1 if an old kernel differs or is missing.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def sass(obj: str) -> dict:
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        if cur is None:
            continue
        line = re.sub(r"/\*[0-9a-f]{4}\*/", "", line)
        line = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", line).strip()
        if line:
            funcs[cur].append(line)
    return funcs


def _name(mangled: str) -> str:
    """_ZN4serl17tgemm_tf32_kernelENS_6TgArgsE -> _ZN4serl17tgemm_tf32_kernel"""
    m = re.match(r"(_ZN4serl(\d+))", mangled)
    return mangled[:m.end() + int(m.group(2))] if m else mangled


def compile_obj(tree: str, src: str, out_dir: str) -> str:
    from serl_b200.build import FLAGS, NVCC
    obj = os.path.join(out_dir, f"{abs(hash(tree))}_{src[:-3]}.o")
    flags = [f.replace(os.path.dirname(HERE), tree) if isinstance(f, str) else f for f in FLAGS]
    subprocess.run([NVCC, *flags, "-c", os.path.join(tree, "serl_b200", "csrc", src), "-o", obj], check=True)
    return obj


def main():
    old_tree, new_tree, srcs = os.path.abspath(sys.argv[1]), os.path.abspath(sys.argv[2]), sys.argv[3:]
    bad = False
    with tempfile.TemporaryDirectory() as tmp:
        for src in srcs:
            a, b = (sass(compile_obj(tree, src, tmp)) for tree in (old_tree, new_tree))
            same, diff, matched = [], [], set()
            for k, body in a.items():
                nk = k if k in b else next((n for n in b if n.startswith(k) or n.startswith(_name(k) + "ILb0E")), None)
                if nk is None:
                    diff.append(k + " (missing)")
                    continue
                matched.add(nk)
                (same if b[nk] == body else diff).append(k)
            new = sorted(set(b) - matched)
            print(f"{src}: {len(same)} kernels with unchanged SASS, {len(diff)} changed, {len(new)} new")
            for k in diff:
                print(f"  changed: {k}")
            for k in new:
                print(f"  new: {k}")
            bad |= bool(diff)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
