"""Tool (not a test): per-kernel SASS comparison of two builds of libnpair_b200.so -- proves that a refactor or an added opt-in
   kernel leaves every existing kernel's machine code untouched.
   python tests/sass_diff.py /path/to/old/libnpair_b200.so [new.so]"""
import hashlib, os, re, subprocess, sys

def funcs(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    d, cur, buf = {}, None, []
    for l in out.split("\n"):
        m = re.match(r"\s*Function : (\S+)", l)
        if m:
            if cur: d[cur] = hashlib.md5("\n".join(buf).encode()).hexdigest()
            cur, buf = m.group(1), []
        elif cur and l.lstrip().startswith("/*"):
            # instruction and encoding lines only, blanks collapsed: cuobjdump pads the instruction column to the widest instruction
            # of the object, and the headers between objects follow the last kernel of each, so neither may depend on the object
            buf.append(" ".join(l.split()))
    if cur: d[cur] = hashlib.md5("\n".join(buf).encode()).hexdigest()
    return d

if __name__ == "__main__":
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    old = funcs(sys.argv[1])
    new = funcs(sys.argv[2] if len(sys.argv) > 2 else os.path.join(here, "npairloss_b200", "lib", "libnpair_b200.so"))
    print(f"{len(old)} kernels before, {len(new)} after")
    print("changed:", [k for k in old if k in new and old[k] != new[k]])
    # a renamed kernel (e.g. an added defaulted template parameter) shows up as removed + new with the same body
    new_only = {k: v for k, v in new.items() if k not in old}
    removed = {k: v for k, v in old.items() if k not in new}
    renamed = [(k, k2) for k, v in removed.items() for k2, v2 in new_only.items() if v == v2]
    print("renamed, identical body:", len(renamed))
    print("removed without an identical successor:", [k for k in removed if k not in [a for a, _ in renamed]])
    print("new    :", [k for k in new_only if k not in [b for _, b in renamed]])
