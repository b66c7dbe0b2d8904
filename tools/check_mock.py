"""Diffs every `//@ref <file>:<first>-<last>` block of serenedb_b200/host/irs_mock.hpp against the cited lines of the
reference tree: each block's declarations (comments and whitespace stripped) must appear, in order, in those lines.
Exit code 0 = the mock's tagged surface is the reference's. Usage: check_mock.py <SereneDB source tree>"""
import os, re, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def strip(text):
    text = re.sub(r"//[^\n]*", "", text)
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"\s+", "", text)


def statements(text):
    """Declarations of a block as whitespace-free token strings, split at ';' '{' '}' (order preserved)."""
    flat = strip(text)
    return [p for p in re.split(r"[;{}]", flat) if p]


def check(ref_root, mock_path=os.path.join(ROOT, "serenedb_b200", "host", "irs_mock.hpp")):
    src = open(mock_path).read()
    blocks = re.findall(r"//@ref (\S+):(\d+)-(\d+)\n(.*?)//@end", src, flags=re.S)
    problems, n_decl = [], 0
    for path, first, last, body in blocks:
        full = os.path.join(ref_root, path)
        if not os.path.exists(full):
            problems.append("%s: missing in the reference tree" % path)
            continue
        lines = open(full).read().split("\n")
        ref = strip("\n".join(lines[max(0, int(first) - 1): int(last)]))
        pos = 0
        for st in statements(body):
            n_decl += 1
            at = ref.find(st, pos)
            if at < 0:
                problems.append("%s:%s-%s: not in the cited lines (or out of order): %s" % (path, first, last, st[:90]))
            else:
                pos = at + len(st)
    return len(blocks), n_decl, problems


if __name__ == "__main__":
    ref_root = sys.argv[1]
    nb, nd, problems = check(ref_root)
    for p in problems:
        print("MISMATCH", p)
    print("%d tagged blocks, %d declarations checked, %d mismatches" % (nb, nd, len(problems)))
    sys.exit(1 if problems else 0)
