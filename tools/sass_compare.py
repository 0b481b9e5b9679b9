"""Check that two trees compile every CUDA kernel to the same machine code.

    python tools/sass_compare.py [--base REV]

Builds the library of REV (default HEAD, checked out with `git worktree` into a temporary directory) and of the
working tree with e4s_b200/build.py's build(force=True), then compares them kernel by kernel:
- the SASS text of every function in every object (cuobjdump -sass), instruction by instruction;
- the registers, shared memory, stack and spills ptxas reported for it (_obj/ptxas.log).
Kernels are matched by demangled name after rename() maps names of the base tree to those of the working tree; every
other name must be present in both.  Exits non-zero on any difference.  nvcc cross-compiles: no GPU needed.
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_BIN = os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"))

# conv3x3_rs_kernel<NT, RES, DENSE, REFL, PW, VOL, CONVT, EPI, ROWS> -> <NT, RES, MODE> (the Mode values of
# csrc/wgmma_conv.cuh), and its CONVT / ROWS instantiations -> the kernels they became.
_RS_MODES = {  # (DENSE, REFL, PW, VOL, EPI) -> MODE
    ("0", "0", "0", "0", "0"): 3,    # FWD_RS
    ("1", "0", "0", "0", "0"): 5,    # FWD_DENSE
    ("1", "1", "0", "0", "0"): 6,    # FWD_REFL
    ("1", "0", "1", "0", "0"): 7,    # FWD_PW
    ("1", "0", "0", "1", "0"): 8,    # FWD_VOL
    ("1", "0", "0", "0", "2"): 9,    # FWD_SPADE
    ("1", "0", "1", "0", "1"): 10,   # FWD_PWF
}
_RS_OLD = re.compile(r"conv3x3_rs_kernel<\(int\)(\d+), \(bool\)(\d), \(bool\)(\d), \(bool\)(\d), \(bool\)(\d), "
                     r"\(bool\)(\d), \(bool\)(\d), \(int\)(\d), \(bool\)(\d)>")


def rename(name: str) -> str:
    m = _RS_OLD.search(name)
    if not m:
        return name
    nt, res, dense, refl, pw, vol, convt, epi, rows = m.groups()
    if convt == "1":
        new = f"convt_rs_kernel<(bool){res}>"
    elif rows == "1":
        new = f"rows_rs_kernel<(int){nt}>"
    else:
        new = f"conv3x3_rs_kernel<(int){nt}, (bool){res}, (int){_RS_MODES[(dense, refl, pw, vol, epi)]}>"
    return name[:m.start()] + new + name[m.end():]


def build_tree(root: str) -> str:
    """build(force=True) of the tree at root, in a child process (the build module of that tree); returns its _obj."""
    code = ("import importlib.util\n"
            "s = importlib.util.spec_from_file_location('b', 'e4s_b200/build.py')\n"
            "m = importlib.util.module_from_spec(s); s.loader.exec_module(m); m.build(force=True)\n")
    subprocess.run([sys.executable, "-c", code], cwd=root, check=True)
    return os.path.join(root, "e4s_b200", "csrc", "_obj")


def demangle(names):
    names = list(names)
    if not names:
        return {}
    out = subprocess.run([os.path.join(CUDA_BIN, "cu++filt")], input="\n".join(names), capture_output=True, text=True,
                         check=True).stdout.splitlines()
    return dict(zip(names, out))


def sass(objdir: str) -> dict:
    """{demangled function: SASS text} over every object in objdir (each name must be defined once); prints how many
    functions each object holds."""
    funcs, counts = {}, []
    for obj in sorted(os.listdir(objdir)):
        if not obj.endswith(".o"):
            continue
        text = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-sass", os.path.join(objdir, obj)],
                              capture_output=True, text=True, check=True).stdout
        name = None
        for line in text.splitlines():
            m = re.match(r"\s*Function : (\S+)", line)
            if m:
                name = m.group(1)
                if name in funcs:
                    raise SystemExit(f"{name} defined twice")
                funcs[name] = []
            elif name and line.strip().startswith("/*"):     # instruction lines: address, text, encoding
                funcs[name].append(" ".join(line.split()))     # (the column padding follows the object's widest line)
        counts.append(f"{obj} {text.count('Function : ')}")
    print("  " + ", ".join(counts))
    dm = demangle(funcs)
    return {dm[k]: "\n".join(v) for k, v in funcs.items()}


def resources(objdir: str) -> dict:
    """{demangled function: ptxas resource lines} from objdir/ptxas.log (build.py writes it with -Xptxas -v)."""
    res, name = {}, None
    with open(os.path.join(objdir, "ptxas.log")) as f:
        for line in f:
            m = re.search(r"(?:Compiling entry function '|Function properties for )([^' ]+)", line)
            if m:
                name = m.group(1).strip()
                res.setdefault(name, [])
            elif name and ("Used" in line or "spill" in line or "stack" in line):
                res[name].append(line.split(":", 1)[-1].strip())
    dm = demangle(res)
    return {dm[k]: v for k, v in res.items()}


def compare(base_obj: str, new_obj: str) -> int:
    failures = 0
    for what, get in (("SASS", sass), ("ptxas resources", resources)):
        print(f"{what}:")
        old = {rename(k): v for k, v in get(base_obj).items()}
        new = get(new_obj)
        same = sum(1 for k in new if k in old and old[k] == new[k])
        print(f"  {len(old)} functions before, {len(new)} after, {same} identical")
        for k in sorted(set(old) - set(new)):
            print(f"  only before: {k}")
            failures += 1
        for k in sorted(set(new) - set(old)):
            print(f"  only after:  {k}")
            failures += 1
        for k in sorted(set(old) & set(new)):
            if old[k] != new[k]:
                print(f"  differs:     {k}")
                failures += 1
    print("identical" if not failures else f"{failures} differences")
    return failures


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--base", default="HEAD", help="revision to compare the working tree against")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="sass_compare_") as tmp:
        base = os.path.join(tmp, "base")
        subprocess.run(["git", "-C", ROOT, "worktree", "add", "--detach", base, args.base], check=True,
                       capture_output=True)
        try:
            base_obj = build_tree(base)
            new_obj = build_tree(ROOT)
            return 1 if compare(base_obj, new_obj) else 0
        finally:
            subprocess.run(["git", "-C", ROOT, "worktree", "remove", "--force", base], check=True)


if __name__ == "__main__":
    sys.exit(main())
