"""Compare the device code of two builds of libb200promql.so, kernel by kernel.

    python profiles/compare_sass.py OLD.so NEW.so

A refactor of the host runtime must leave every kernel as it was.  This maps each kernel's demangled name to its SASS
instruction stream (cuobjdump -sass; the /*addr*/ column is dropped and white space collapsed, the encodings with their
scheduling bits are kept) and to its resource usage (cuobjdump -res-usage: registers, shared memory, stack, ...), and checks that both builds
have the same kernels with the same streams and resources.  Two things depend on the module a kernel is in, not on the
kernel, and are not compared: the slot of a global's address in the symbol bank c[0x4] (masked, with that word's
encoding), and the 1 KB of system-reserved shared memory sm_90 reports for every kernel of a module that uses it
(counted and printed).  A kernel that now appears in several modules (a CUB
template instantiated by more than one translation unit) must have one stream, equal to the old one, in all of them.
Exit status 0 when everything matches.
"""
import collections
import re
import subprocess
import sys

CUDA = "/usr/local/cuda/bin/"


def demangle(names):
    out = subprocess.run([CUDA + "cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, out.stdout.splitlines()))


def sass(lib):
    """{mangled name: set of instruction streams}"""
    text = subprocess.run([CUDA + "cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs = collections.defaultdict(set)
    name, body = None, []
    for line in text.splitlines() + ["\t\tFunction : <end>"]:
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name].add("\n".join(body))
            name, body = m.group(1), []
        elif not line.startswith((" ", "\t")):  # the header of the next module's fatbin ends the function
            if name:
                funcs[name].add("\n".join(body))
            name, body = None, []
        elif name and line.strip() and not line.strip().startswith((".headerflags", "..........")):
            ins = " ".join(re.sub(r"^\s*/\*[0-9a-f]{4,}\*/", "", line).split())
            if "c[0x4][" in ins:  # the address of a global in the module's symbol bank: its slot depends on the module
                ins = re.sub(r"c\[0x4\]\[[^\]]*\]", "c[0x4][sym]", ins.split(" /*")[0])
            body.append(ins)
    funcs.pop("<end>", None)
    return funcs


def resources(lib):
    """{mangled name: set of resource lines}"""
    text = subprocess.run([CUDA + "cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    res = collections.defaultdict(set)
    name = None
    for line in text.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            res[name].add(line.strip())
            name = None
    return res


def main(old, new):
    s_old, s_new = sass(old), sass(new)
    r_old, r_new = resources(old), resources(new)
    names = demangle(sorted(set(s_old) | set(s_new)))
    ok = True
    if set(s_old) != set(s_new):
        ok = False
        for n in sorted(set(s_old) - set(s_new)):
            print("only in old:", names[n])
        for n in sorted(set(s_new) - set(s_old)):
            print("only in new:", names[n])
    diff_sass = [n for n in set(s_old) & set(s_new) if len(s_new[n]) != 1 or s_new[n] != s_old[n]]
    diff_res, reserved = [], []
    for n in set(r_old) | set(r_new):
        if r_old.get(n) == r_new.get(n):
            continue
        a, b = (re.sub(r"SHARED:\d+", "", next(iter(r.get(n, {""})))) for r in (r_old, r_new))
        shared = [int(m) for r in (r_old, r_new) for m in re.findall(r"SHARED:(\d+)", next(iter(r.get(n, {""}))))]
        # sm_90 reports the 1 KB of system-reserved shared memory per CTA for every kernel of a module where some
        # kernel uses it; a module without such a kernel reports none.  The launch reserves it either way.
        if a == b and len(shared) == 2 and abs(shared[0] - shared[1]) == 1024 and len(r_new[n]) == 1:
            reserved.append(n)
        else:
            diff_res.append(n)
    for n in sorted(diff_sass):
        print("instruction stream differs:", names[n])
    for n in sorted(diff_res):
        print("resource usage differs:", names.get(n, n), r_old.get(n), r_new.get(n))
    if reserved:
        print(f"{len(reserved)} kernels differ only in the module's 1 KB of reserved shared memory (SHARED +-1024)")
    ok = ok and not diff_sass and not diff_res
    copies = sum(len(v) for v in s_new.values())
    print(f"{len(s_old)} kernels in old, {len(s_new)} in new; "
          f"{sum(1 for n in s_new if len(s_new[n]) == 1)} with one distinct stream in new; "
          f"{len(diff_sass)} streams differ, {len(diff_res)} resource usages differ -> {'SAME' if ok else 'DIFFERENT'}")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1], sys.argv[2]))
