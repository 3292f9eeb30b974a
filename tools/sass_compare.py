"""Compare the SASS of the kernels two object files share, instruction by instruction (the encodings included), with the
mangled names reduced to the kernel template and its task: a changed source must leave the listed kernels bit-identical.

    python tools/sass_compare.py parent/episode_kernels.o episode_kernels.o [--match continuous]

Builds nothing: compile both objects with the Makefile's flags first (nvcc ... -c episode_kernels.cu -o ...).  A kernel
whose template gained a parameter is matched by its name and task with the new parameter's default mode (`Lb0E`: false).
Exits 1 when a matched kernel differs or is missing from the second object."""
import argparse
import re
import subprocess
import sys


def functions(obj: str) -> dict:
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    fs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fs[cur] = []
        elif cur is not None and "/* 0x" in line:
            fs[cur].append(re.sub(r"/\*[0-9a-f]{4}\*/", "", line).strip())     # the address is not the code
    return fs


def short(name: str) -> str:
    m = re.match(r"_Z\d+(\w+?)I(\d+)(\w+?)(Lb[01]E)?E?v", name)
    if not m:
        return name
    task = m.group(3)[:int(m.group(2))]
    return f"{m.group(1)}<{task}{', ' + m.group(4)[2] if m.group(4) else ''}>"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--match", default="continuous", help="compare the kernels whose mangled name contains this")
    a = ap.parse_args()
    old = {short(n): v for n, v in functions(a.old).items() if a.match in n}
    new = {short(n): v for n, v in functions(a.new).items() if a.match in n}
    bad = 0
    for k, v in sorted(old.items()):
        w = new.get(k) if k in new else new.get(k[:-1] + ", 0>")
        same = w == v
        bad += not same
        print(f"{k}: {len(v)} lines, {'identical' if same else 'MISSING' if w is None else 'DIFFERENT'}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
