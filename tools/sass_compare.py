"""Compares the SASS of kernels in two builds (objects or shared libraries), ignoring register numbering (with the
operand-reuse flags that follow it), the offsets of kernel parameters in the constant bank and the hash nvcc gives a
file's anonymous namespace (it changes with any edit to the file): a refactor that must not change what a kernel
executes passes.

    python tools/sass_compare.py OLD.o NEW.o [KERNEL_REGEX ...]

Prints one line per kernel (same / DIFFERENT / missing) and exits 1 when any compared kernel differs."""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
_REG = re.compile(r"\b(U?R\d+|U?P[0-6])\b")
_CBANK = re.compile(r"c\[0x0\]\[0x[0-9a-f]+\]")
_ADDR = re.compile(r"/\*[0-9a-f]{4,}\*/")
_ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_")


def kernels(path):
    out = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = _ANON.sub("_GLOBAL__N__", m.group(1))
            funcs[name] = []
            continue
        if name and "/*" in line and ";" in line:
            ins = _ADDR.sub("", line.split(";")[0]).replace(".reuse", "")
            funcs[name].append(" ".join(_CBANK.sub("c[bank]", _REG.sub("r", ins)).split()))
    return funcs


def main(argv):
    if len(argv) < 3:
        sys.exit(__doc__)
    old, new = kernels(argv[1]), kernels(argv[2])
    pats = [re.compile(p) for p in argv[3:]] or [re.compile(".")]
    bad = 0
    for name in sorted(set(old) | set(new)):
        if not any(p.search(name) for p in pats):
            continue
        if name not in old or name not in new:
            print(f"missing in {'old' if name not in old else 'new'}: {name}")
            bad += 1
        elif old[name] != new[name]:
            print(f"DIFFERENT ({len(old[name])} -> {len(new[name])} instructions): {name}")
            bad += 1
        else:
            print(f"same ({len(new[name])} instructions): {name}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main(sys.argv)
