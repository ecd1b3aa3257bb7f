"""Compare the SASS of every kernel of one build of libbbb_b200.so with the same kernel in another, e.g. the library of
a parent commit against the working tree's, to show that a change leaves existing instantiations' code as it was.

    python tools/sass_diff.py OLD.so NEW.so

A kernel template that gained a trailing flag (<a, b> -> <a, b, false>), or a kernel that gained a trailing
PriorPtrs parameter, is matched to that instantiation.  Prints SAME / DIFF per kernel of OLD.so (instruction words,
addresses stripped) and the kernels only NEW.so has; exits 1 if any kernel of OLD.so differs or is missing."""
import collections
import re
import subprocess
import sys


def kernels(so):
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    fs, cur = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fs[cur] = []
        elif cur is not None:
            # (runs of blanks collapsed: cuobjdump pads every line to the widest instruction of the whole library, so a
            # kernel that gains a longer instruction would shift the columns of every other one)
            ins = re.sub(r"\s+", " ", re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)).strip()
            if ins:
                fs[cur].append(ins)
    return fs


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    dold, dnew = demangle(list(old)), demangle(list(new))
    by_name = {v: k for k, v in dnew.items()}
    bad, matched = 0, set()
    for k, ins in old.items():
        dm = dold[k]
        cands = [dm]
        m = re.match(r"(.*?)<(.*)>\((.*)\)$", dm)
        if m:
            cands += [f"{m.group(1)}<{m.group(2)}, false>({m.group(3)})",
                      f"{m.group(1)}<{m.group(2)}, false>({m.group(3)}, bbb::PriorPtrs)"]
        nk = next((by_name[c] for c in cands if c in by_name), None)
        if nk is None:
            print("MISSING", dm)
            bad += 1
            continue
        matched.add(nk)
        same = ins == new[nk]
        bad += not same
        print(f"{'SAME' if same else 'DIFF'} {len(ins):6d} lines  {dm}" + ("" if dm == dnew[nk] else f"  ->  {dnew[nk]}"))
    print(f"{len(old)} kernels in {sys.argv[1]}: {bad} differ or are missing")
    for k in new:
        if k not in matched:
            print("NEW", dnew[k])
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
