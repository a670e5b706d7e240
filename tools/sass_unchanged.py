"""Check that every kernel (and device function) of a base revision's libwva_b200.so compiles to the same SASS in the
working tree's library.  Needs nvcc and cuobjdump, no GPU.

    python tools/sass_unchanged.py --base REV [--lib inferno-autoscaler_b200/libwva_b200.so]

REV is the revision to compare against: the parent of a committed change (`--base HEAD^`), or `--base HEAD` for
uncommitted work in the tree.  There is no default: comparing a commit with itself would always pass.

The base revision's sources are exported with `git archive` into a temporary directory and compiled with the flags of
__graft_entry__.build_cuda.  Functions that exist only in the working tree (new kernels) are listed, not compared.
Exit status 0 when every base function is byte-identical in the SASS listing, 1 otherwise.
"""
import argparse
import io
import os
import re
import subprocess
import sys
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

CUOBJDUMP = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")


def functions(lib):
    """{mangled name: SASS text} of every function in the library's sm_90a cubin"""
    out = subprocess.check_output([CUOBJDUMP if os.path.exists(CUOBJDUMP) else "cuobjdump", "-sass", lib], text=True)
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = "\n".join(body)
            name, body = m.group(1), []
        elif name is not None:
            body.append(line)
    if name:
        funcs[name] = "\n".join(body)
    return funcs


def build_base(rev, outdir):
    data = subprocess.check_output(["git", "-C", ROOT, "archive", rev, "include", "inferno-autoscaler_b200/csrc"])
    tarfile.open(fileobj=io.BytesIO(data)).extractall(outdir)
    csrc = os.path.join(outdir, "inferno-autoscaler_b200", "csrc")
    lib = os.path.join(outdir, "libwva_b200.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + graft.NVCC_FLAGS + ["-o", lib, os.path.join(csrc, "wva_b200.cu")], cwd=csrc,
                          stderr=subprocess.DEVNULL)
    return lib


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--base", required=True, help="git revision to compare against (e.g. HEAD^ for a committed change)")
    ap.add_argument("--lib", default=graft.LIB, help="library of the working tree (built when missing)")
    args = ap.parse_args()
    if not os.path.exists(args.lib):
        graft.build_cuda()
    with tempfile.TemporaryDirectory() as tmp:
        base = functions(build_base(args.base, tmp))
    new = functions(args.lib)
    changed = [f for f in sorted(base) if new.get(f) != base[f]]
    added = sorted(set(new) - set(base))
    print("base %s: %d functions; working tree: %d functions" % (args.base, len(base), len(new)))
    print("added: %s" % (", ".join(added) if added else "none"))
    for f in changed:
        print("CHANGED: %s%s" % (f, " (missing)" if f not in new else ""))
    print("every base function identical" if not changed else "%d base functions differ" % len(changed))
    return 1 if changed else 0


if __name__ == "__main__":
    sys.exit(main())
