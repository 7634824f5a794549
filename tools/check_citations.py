"""Checks that every reference citation of the form `<path>.py:<line>[-<line>]` in the repo's sources and docs names a
file that exists under /root/reference (SpeechT5 tree first, sibling trees second) and a line range inside it. Runs
only where the reference is mounted (this container); prints the broken ones and exits 1 if any.
usage: python tools/check_citations.py [-v]"""
import glob
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ST5_REFERENCE_ROOT", "/root/reference")  # the same root as oracle/ref_loader.py
ALIAS = {"legacy_ddp.py": "fairseq/distributed/legacy_distributed_data_parallel.py"}  # SURVEY.md:15 shorthand
PAT = re.compile(r"([A-Za-z0-9_./-]+\.py):(\d+)(?:-(\d+))?")


def index():
    by_tail = {}
    for p in glob.glob(REF + "/**/*.py", recursive=True):
        rel = p[len(REF) + 1:]
        parts = rel.split("/")
        for i in range(len(parts)):
            by_tail.setdefault("/".join(parts[i:]), []).append(p)
    return by_tail


def main():
    verbose = "-v" in sys.argv
    if not os.path.isdir(REF):
        print("reference not mounted; nothing checked")
        return 0
    by_tail = index()
    files = [p for pat in ("*.md", "include/*.h", "oracle/*.py", "speecht5_b200/**/*.py", "speecht5_b200/csrc/*",
                           "tests/**/*.py", "bench.py", "__graft_entry__.py")
             for p in glob.glob(os.path.join(ROOT, pat), recursive=True)]
    lens, bad, n = {}, [], 0
    for f in sorted(set(files)):
        if os.path.basename(f) in ("SURVEY.md", "PAPERS.md", "SNIPPETS.md", "BASELINE.md", "VERDICT.md", "ADVICE.md"):
            continue
        for ln, line in enumerate(open(f, errors="ignore"), 1):
            for m in PAT.finditer(line):
                path, a, b = m.group(1), int(m.group(2)), int(m.group(3) or m.group(2))
                if "..." in path:
                    continue
                path = path.lstrip("./")
                if path.startswith("root/reference/"):
                    path = path[len("root/reference/"):]
                path = ALIAS.get(path, path)
                if os.path.exists(os.path.join(ROOT, path)):  # a citation of this repo's own file
                    continue
                cands = by_tail.get(path)
                if not cands:
                    bad.append((f, ln, m.group(0), "no such reference file"))
                    continue
                n += 1
                cands = sorted(cands, key=lambda p: (0 if "/SpeechT5/" in p else 1, len(p)))
                ok = False
                for c in cands:
                    if c not in lens:
                        lens[c] = sum(1 for _ in open(c, errors="ignore"))
                    if a <= b <= lens[c]:
                        ok = True
                        break
                if not ok:
                    bad.append((f, ln, m.group(0), f"line range outside the file ({lens[cands[0]]} lines)"))
                elif verbose:
                    print("ok", m.group(0))
    for f, ln, cite, why in bad:
        print(f"{f[len(ROOT) + 1:]}:{ln}: {cite}: {why}")
    print(f"{n} citations checked, {len(bad)} broken")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
