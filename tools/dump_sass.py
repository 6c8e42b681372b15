"""Per-kernel SASS listings under profiles/sass/ (git-ignored): one file per kernel family (first
template instantiation of each, plus the named flagship instantiations), and an index with the
Hopper-relevant mnemonic counts of EVERY instantiation (HGMMA = wgmma, WARPGROUP = its
fences, UTMALDG/UTMASTG = TMA, LDGMC = multimem.ld_reduce, HMMA would be the legacy path)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "veles", "znicz_b200", "kernels", "_znicz_b200_C.so")
OUT = os.path.join(ROOT, "profiles", "sass")
MNEMONICS = ("HGMMA", "WARPGROUP", "USETMAXREG", "UTMALDG", "UTMASTG", "UBLKCP", "LDGSTS",
             "LDGMC", "STGMC", "REDGMC", "UCGABAR", "SYNCS", "HMMA", "FFMA", "MUFU", "ATOM", "RED.")
KEEP_EXTRA = ("gemm_pair_k<256, false>", "gemm_pair_k<(int)256, (bool)0>")


def demangle(names):
    p = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return p.stdout.splitlines()


def main():
    txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
    funcs = []
    cur = None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = [m.group(1), []]
            funcs.append(cur)
        elif cur is not None:
            cur[1].append(line)
    names = demangle([f[0] for f in funcs])
    os.makedirs(OUT, exist_ok=True)
    for f in os.listdir(OUT):
        os.remove(os.path.join(OUT, f))
    seen = {}
    index = []
    for (mangled, body), name in zip(funcs, names):
        fam = re.sub(r"^void ", "", name).split("<")[0].split("(")[0].replace("zn::", "")
        fam = re.sub(r"[^A-Za-z0-9_]+", "_", fam).strip("_")
        code = [l for l in body if re.search(r"/\*[0-9a-f]{4,}\*/", l)]
        counts = collections.Counter()
        for l in code:
            for mn in MNEMONICS:
                if mn in l:
                    counts[mn] += 1
        index.append((fam, name, len(code), counts))
        if fam not in seen or any(k in name for k in KEEP_EXTRA):
            fn = fam if fam not in seen else fam + "_flagship"
            seen.setdefault(fam, fn)
            with open(os.path.join(OUT, fn + ".sass"), "w") as out:
                out.write("// %s\n// (%d instructions; cuobjdump -sass of the in-tree "
                          "_znicz_b200_C.so, sm_90a)\n" % (name, len(code)))
                # strip the encoding column: keeps the listing readable and ~3x smaller
                for l in code:
                    out.write(re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", l).rstrip() + "\n")
    with open(os.path.join(OUT, "INDEX.md"), "w") as out:
        out.write("# SASS index (tools/dump_sass.py; sm_90a, %d kernels)\n\n" % len(index))
        out.write("| family | instantiation | instr | " + " | ".join(MNEMONICS) + " |\n")
        out.write("|---|---|---|" + "---|" * len(MNEMONICS) + "\n")
        for fam, name, n, c in sorted(index):
            short = name if len(name) < 110 else name[:107] + "..."
            out.write("| %s | `%s` | %d | %s |\n" % (
                fam, short.replace("|", "/"), n, " | ".join(str(c.get(m, 0) or "") for m in MNEMONICS)))
    print("wrote %d listings, %d kernels indexed" % (len(seen), len(index)))


if __name__ == "__main__":
    sys.exit(main())
