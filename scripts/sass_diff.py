"""Compare the compiled kernels of a git revision with those of the working tree, function by function.

    python scripts/sass_diff.py                  # HEAD against the working tree
    python scripts/sass_diff.py --base HEAD~1    # the last commit's parent against the working tree

Both trees compile the kernel sources in SOURCES through the library's Makefile, with the build's flags, into
temporary directories; nothing in the repository is written.  A source the base does not have is compiled from the
working tree alone and its functions are listed as new.  Functions are matched by their demangled name without the
parameter list (cu++filt), so that a kernel whose arguments moved into a struct is still compared with itself, and their
SASS with runs of spaces collapsed, since cuobjdump pads every line to the widest instruction of the file.  The script
prints every function whose SASS is not byte-identical, with its instruction count before and after, and fails (exit
status 1) when a function appears or disappears, or when anything ptxas -v reports differs from the base: a function's
registers, barriers, shared and constant memory, stack frame, spills or diagnostics (counted by code), or the
file-wide totals."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join("metal-flash-attention_b200", "csrc")
SOURCES = ("kernels/wgmma_attention.cu", "kernels/simt_attention.cu", "kernels/paged_append.cu",
           "kernels/rotary_append.cu")
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
CUFILT = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cu++filt")


def compile_tree(tree, out):
    """Object files of the SOURCES `tree` has, compiled from its Makefile into `out`: {source: (object, ptxas log)}"""
    present = [src for src in SOURCES if os.path.exists(os.path.join(tree, CSRC, src))]
    objs = [os.path.join(out, src.replace(".cu", ".o")) for src in present]
    subprocess.check_call(["make", "-s", "-j", str(len(objs)), "-C", os.path.join(tree, CSRC), f"BUILD={out}", *objs])
    return {src: (obj, obj + ".ptxas.log") for src, obj in zip(present, objs)}


def anonymous(text):
    """text with each anonymous namespace's per-compilation id removed: nvcc derives it from the compilation, so the
    same source compiled in two trees names its functions differently"""
    return re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", text)


def without_parameters(demangled):
    """a demangled function name without its trailing parameter list"""
    if not demangled.endswith(")"):
        return demangled
    depth = 0
    for i in range(len(demangled) - 1, -1, -1):
        depth += {")": 1, "(": -1}.get(demangled[i], 0)
        if depth == 0:
            return demangled[:i]
    return demangled


def keys(names):
    """{mangled name: the key a function is matched by}; fails if two functions of one file share a key"""
    names = sorted(set(names))
    out = subprocess.run([CUFILT], input="\n".join(names) + "\n", capture_output=True, text=True, check=True).stdout
    key = {name: without_parameters(d) for name, d in zip(names, out.splitlines())}
    if len(set(key.values())) != len(key):
        sys.exit("sass_diff: two functions share a name without their parameter lists")
    return key


def sass(obj):
    """{function key: SASS text} of an object file, runs of spaces collapsed"""
    text = anonymous(subprocess.check_output([CUOBJDUMP, "-sass", obj], text=True))
    funcs, name = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(re.sub(" +", " ", line))  # (cuobjdump pads to the widest line of the whole file)
    key = keys(funcs)
    return {key[name]: "\n".join(lines) for name, lines in funcs.items()}


def instructions(text):
    return sum(1 for line in text.splitlines() if re.match(r"\s*/\*[0-9a-f]{4,}\*/", line))


def ptxas_report(log):
    """{function key: what ptxas -v reported for it} -- its resource line (registers, barriers, smem, cmem), its stack and
    spill line, and how many diagnostics of each code it drew (without their PTX line numbers, which move with any
    source edit).  Key None holds the lines that belong to no function, such as the gmem total."""
    report, name = {None: {}}, None
    with open(log) as f:
        for line in map(anonymous, f):
            text = line.split(":", 1)[-1].strip()
            m = re.search(r"Compiling entry function '(\S+)'|Function properties for (\S+)", line)
            if m:
                name = m.group(1) or m.group(2)
                report.setdefault(name, {})
            elif d := re.search(r"\((C\d+)\).* in function '(\S+)'", line):
                code, func = d.groups()
                entry = report.setdefault(func, {})
                entry[code] = entry.get(code, 0) + 1
            elif text.startswith("Used "):
                report[name]["resources"] = text
            elif "bytes stack frame" in text:
                report[name]["stack and spills"] = text
            elif text and not text.startswith("Compile time"):
                report[None][text] = report[None].get(text, 0) + 1
    key = keys(name for name in report if name is not None)
    return {key.get(name): entry for name, entry in report.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default="HEAD", help="git revision to compare the working tree against (default HEAD)")
    args = ap.parse_args()
    ok = True
    with tempfile.TemporaryDirectory() as tmp:
        base_tree = os.path.join(tmp, "base")
        os.makedirs(base_tree)
        archive = subprocess.check_output(["git", "-C", ROOT, "archive", args.base])
        subprocess.run(["tar", "-x", "-C", base_tree], input=archive, check=True)
        before = compile_tree(base_tree, os.path.join(tmp, "build_base"))
        after = compile_tree(ROOT, os.path.join(tmp, "build_tree"))
        for src in SOURCES:
            if src not in before:
                print(f"{src}: new in the working tree, {len(sass(after[src][0]))} functions")
                continue
            (obj_a, log_a), (obj_b, log_b) = before[src], after[src]
            sa, sb = sass(obj_a), sass(obj_b)
            ra, rb = ptxas_report(log_a), ptxas_report(log_b)
            same = [f for f in sa if f in sb and sa[f] == sb[f]]
            print(f"{src}: {len(sa)} functions in {args.base}, {len(sb)} in the working tree, {len(same)} byte-identical")
            for f in sorted(set(sa) ^ set(sb)):
                print(f"  only in {args.base if f in sa else 'the working tree'}: {f}")
                ok = False
            for f in sorted(set(sa) & set(sb)):
                if sa[f] != sb[f]:
                    print(f"  SASS differs: {f}: {instructions(sa[f])} -> {instructions(sb[f])} instructions")
            for f in sorted(set(ra) | set(rb), key=str):
                if ra.get(f) != rb.get(f):
                    print(f"  PTXAS REPORT differs: {f or 'outside any function'}: {ra.get(f)} -> {rb.get(f)}")
                    ok = False
    print("resources unchanged" if ok else "FAILED")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
