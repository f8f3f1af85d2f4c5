"""Counts a kernel's local-memory instructions (LDL / STL: register spills and local arrays) per source line.

usage: spill_lines.py BINARY [KERNEL ...]
  BINARY: a cubin, or a library / object with sm_90a code in it (brotli_b200/libbrotlienc_b200.so); the cubins are
          extracted with cuobjdump.  Build it with -lineinfo (the product build does), or every line reads as unknown.
  KERNEL: substrings of the kernels' mangled names (default: k_walk), e.g. _Z6k_walkILi1025ELb0E for the quality-5 walker
          (br_walk_form: 1025 = G 1 with a fixed 16-entry ring, 1281 = G 1 with 32 entries, 4 = G 4, 0 = quick search).
For every matching kernel: its instruction count, its LDL and STL counts, then the lines holding local-memory
instructions, most first, as file:line (the innermost source line nvdisasm -g names).  -Xptxas -v gives the spill bytes;
this gives where they sit.
"""
import collections, os, re, subprocess, sys, tempfile

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def disasm(cubin):
    return subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "-g", "-c", cubin], check=True,
                          capture_output=True, text=True).stdout


def cubins(path, tmp):
    if path.endswith(".cubin"):
        return [path]
    subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(path)], cwd=tmp, check=True,
                   capture_output=True)
    return [os.path.join(tmp, f) for f in sorted(os.listdir(tmp)) if f.endswith(".cubin")]


def kernels(text):
    """yields (mangled name, [(source line, opcode)])"""
    name, body, line = None, [], "?"
    for ln in text.splitlines():
        m = re.match(r"^\.text\.(\S+):", ln)
        if m:
            if name:
                yield name, body
            name, body, line = m.group(1), [], "?"
            continue
        m = re.match(r'^\s*//## File "([^"]+)", line (\d+)', ln)
        if m:
            line = "%s:%s" % (os.path.basename(m.group(1)), m.group(2))
            continue
        m = re.match(r"^\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", ln)
        if m and name:
            body.append((line, m.group(1)))
    if name:
        yield name, body


def main():
    if len(sys.argv) < 2:
        sys.exit(__doc__)
    pats = sys.argv[2:] or ["k_walk"]
    with tempfile.TemporaryDirectory() as tmp:
        for cb in cubins(sys.argv[1], tmp):
            for name, body in kernels(disasm(cb)):
                if not any(p in name for p in pats):
                    continue
                per = collections.Counter(l for l, op in body if op.split(".")[0] in ("LDL", "STL"))
                ldl = sum(1 for _, op in body if op.split(".")[0] == "LDL")
                stl = sum(1 for _, op in body if op.split(".")[0] == "STL")
                print("%s: %d instructions, %d LDL, %d STL" % (name, len(body), ldl, stl))
                for l, c in per.most_common():
                    print("  %4d  %s" % (c, l))


if __name__ == "__main__":
    main()
