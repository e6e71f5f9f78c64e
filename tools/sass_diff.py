"""Per-kernel SASS diff of two builds of one object file (development tool, CPU only).

    python tools/sass_diff.py PARENT/evo_b200/build/hyena.o evo_b200/build/hyena.o

Kernels are keyed by their demangled name without the argument list; a trailing `false` template flag (the RESUME form of
hyena_scan_ms_kernel, the PREFIX form of attn_fwd_kernel, the FP8
form of gemm_smallm_kernel) is dropped, so a pre-existing instantiation lines up with the one
it was before the flag existed.  Compare object files, not the linked library: linking moves global addresses.  Exit code 1
if a pre-existing kernel's SASS changed or disappeared."""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def kernels(path):
    out = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    body, cur, name = {}, [], None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                body[name] = cur
            name, cur = m.group(1), []
        elif name is not None:
            cur.append(re.sub(r"\s+", " ", line.strip()))
    if name:
        body[name] = cur
    names = list(body)
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    res = {}
    for mangled, d in zip(names, dem):
        key = re.sub(r"\((?!anonymous namespace\)).*$", "", d)
        key = re.sub(r"<(true|false), (true|false), false>$", r"<\1, \2>", key)
        if "attn_fwd_kernel" in key:
            key = re.sub(r"<(true|false), false>$", r"<\1>", key)
        if "gemm_smallm_kernel" in key:
            key = re.sub(r", false>$", ">", key)
        res[key] = body[mangled]
    return res


def main(a_path, b_path):
    a, b = kernels(a_path), kernels(b_path)
    diff = [k for k in a if k in b and a[k] != b[k]]
    gone = [k for k in a if k not in b]
    new = [k for k in b if k not in a]
    print(f"{len(a)} kernels before: {len(a) - len(diff) - len(gone)} identical, {len(diff)} different, {len(gone)} missing; {len(new)} new")
    for tag, ks in (("DIFFERENT", diff), ("MISSING", gone), ("NEW", new)):
        for k in ks:
            print(f"  {tag} {k}")
    return 1 if diff or gone else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1], sys.argv[2]))
