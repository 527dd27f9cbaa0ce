"""Compare the SASS of every kernel of two builds of a CUDA object (cubin, .o or .so), e.g. the parent commit's
mvp_kernels.cu and the current one: `cuobjdump -sass` of each, split per function, and the instruction text compared after
dropping the function name and comments.  A kernel template that gained a trailing defaulted parameter is matched through
--suffix (the mangled spelling of that parameter's default, e.g. Lb0E).  Needs no GPU.

    python scripts/sass_identity.py old.cubin new.cubin --suffix Lb0E
Prints one line per kernel of the old build and exits non-zero if any differs or is missing."""
import argparse
import re
import subprocess
import sys


def functions(path):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = body
            # the anonymous namespace's mangled name carries a hash of the translation unit: not part of the comparison
            name, body = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_(\w+?)_[0-9a-f]{8}", r"_GLOBAL__N_\1", m.group(1)), []
        elif name and re.match(r"\s*/\*[0-9a-f]{4,}\*/", line):
            body.append(re.sub(r"\s*/\*[0-9a-f]{4,}\*/\s*", "", line.split(";")[0]).strip() + ";")
    if name:
        funcs[name] = body
    return funcs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--suffix", default="", help="mangled default template argument appended in the new build")
    a = ap.parse_args()
    old, new = functions(a.old), functions(a.new)
    bad = 0
    for name, body in sorted(old.items()):
        cand = [name]
        if a.suffix:
            cand.append(re.sub(r"EEv", a.suffix + "EEv", name, count=1))
        match = next((c for c in cand if c in new), None)
        if match is None:
            print("MISSING   %s" % name)
            bad += 1
            continue
        same = new[match] == body
        bad += not same
        print("%s %5d instr  %s" % ("IDENTICAL" if same else "DIFFERENT", len(body), name))
    print("%d kernels of the old build, %d of the new; %d differ or are missing" % (len(old), len(new), bad))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
