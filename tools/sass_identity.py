"""Function-by-function comparison of the device code (SASS) of two builds of libb200trk.so:

    python tools/sass_identity.py OLD.so NEW.so

Used to prove that moving validated kernels into `*_kernels.cuh` headers (so that the CPU tier can execute them under
tests/cpu_emul/cuda_shim.h) changed no device instruction.  Kernels in anonymous namespaces carry a hash of the build path in their mangled
name; it is masked before matching."""
import re
import subprocess
import sys


def funcs(so):
    txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    txt = "\n".join(l for l in txt.split("\n") if l.strip())
    out = {}
    for p in re.split(r"\n(?=\t\tFunction : )", txt)[1:]:
        name = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_", "_GLOBAL__N__HASH_", p.split("\n", 1)[0].strip().replace("Function : ", ""))
        body = re.split(r"\n(?=Fatbin|\s*\.\.\.\.|code for sm)", p.split("\n", 1)[1])[0].strip()
        # cuobjdump pads its columns to the longest instruction of the whole cubin, so a kernel added to a translation unit re-pads
        # the listing of its unchanged neighbours: compare instructions and encodings, not the padding
        out[name] = re.sub(r"[ \t]+", " ", body)
    return out


def main():
    a, b = funcs(sys.argv[1]), funcs(sys.argv[2])
    same = [k for k in a if k in b and a[k] == b[k]]
    diff = [k for k in a if k in b and a[k] != b[k]]
    gone = [k for k in a if k not in b]
    new = [k for k in b if k not in a]
    print("kernels: %d -> %d | identical %d, different %d, removed %d, new %d" % (len(a), len(b), len(same), len(diff), len(gone), len(new)))
    for tag, ks in (("DIFFERENT", diff), ("REMOVED", gone), ("NEW", new)):
        for k in ks:
            print("%-9s %s" % (tag, k))
    return 1 if diff or gone else 0


if __name__ == "__main__":
    sys.exit(main())
