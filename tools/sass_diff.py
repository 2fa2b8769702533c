"""Compare the SASS of every kernel of a parent build's object with the same kernel of a new build.

    python tools/sass_diff.py OLD.o NEW.o [OLD.o NEW.o ...]

Kernels are matched by name without their argument list.  A kernel that gained a trailing `bool` template parameter (an FMAP or
similar switch whose `false` instantiation is meant to stay the parent's code) is matched by its old name plus `, false`, and a plain
kernel that became a template of one such parameter by its old name plus `<false>`.  Prints one line per kernel of the old object (same / DIFFERENT /
missing) and exits 1 if any is not the same.  Register counts come from `cuobjdump -res-usage`."""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
CUFILT = "/usr/local/cuda/bin/cu++filt"


def demangle(names):
    """mangled -> demangled name without its argument list (a kernel that gained a parameter keeps its name)"""
    out = subprocess.run([CUFILT], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    return {k: d[:d.rfind(">(") + 1] if ">(" in d else d.split("(")[0] for k, d in zip(names, out)}


def sass(obj):
    """{demangled kernel: its SASS instructions, one string}"""
    txt = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur and re.match(r"\s*/\*[0-9a-f]{4,}\*/", line):
            funcs[cur].append(line.strip())
    names = demangle(list(funcs))
    return {names[k]: "\n".join(v) for k, v in funcs.items()}


def regs(obj):
    txt = subprocess.run([CUOBJDUMP, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if cur and m:
            out[cur] = (int(m.group(1)), int(m.group(2)))
    names = demangle(list(out))
    return {names[k]: v for k, v in out.items()}


def with_false(name):
    """k<a, b> -> k<a, b, false>; k -> k<false>"""
    return name[:-1] + ", (bool)0>" if name.endswith(">") else "void %s<(bool)0>" % name


def main(pairs):
    bad = 0
    for old_o, new_o in pairs:
        old, new = sass(old_o), sass(new_o)
        rold, rnew = regs(old_o), regs(new_o)
        same = 0
        for k in sorted(old):
            n = k if k in new else with_false(k)
            if n not in new:
                print("missing    %s" % k)
                bad += 1
            elif old[k] != new[n] or rold.get(k) != rnew.get(n):
                print("DIFFERENT  %s  (regs/stack %s -> %s)" % (k, rold.get(k), rnew.get(n)))
                bad += 1
            else:
                same += 1
        print("%s: %d of %d parent kernels compile to the same SASS, registers and stack in %s" % (old_o, same, len(old), new_o))
    return 1 if bad else 0


if __name__ == "__main__":
    a = sys.argv[1:]
    if not a or len(a) % 2:
        sys.exit(__doc__)
    sys.exit(main(list(zip(a[::2], a[1::2]))))
