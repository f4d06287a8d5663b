"""Compares the SASS of two builds of libmeao.so function by function: `cuobjdump -sass` of each, with the hash-derived parts of the
anonymous-namespace names and the source-path lines normalised away, so a function whose instructions are unchanged compares equal.
Prints one JSON line: the function counts, how many of the first build's functions differ or are missing in the second, and the names.
Used to show that a change which adds kernels leaves the existing ones byte for byte as they were.

    python scripts/sass_diff.py OLD/libmeao.so NEW/libmeao.so
"""
import json
import re
import subprocess
import sys

_ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+")


def functions(lib: str) -> dict:
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    res, name, body = {}, None, []
    for line in _ANON.sub("ANON", out).splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            if name:
                res[name] = body
            name, body = m.group(1), []
        elif name:
            text = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).strip()
            # the container lines between two files' functions and the source path are not the function's code
            if not text.startswith(("identifier =", "Fatbin", "=====", "arch =", "code version", "code for", "host =", "compile_size")):
                body.append(text)
    if name:
        res[name] = body
    return {n: "\n".join(x for x in b if x) for n, b in res.items()}


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    differ = sorted(n for n in old if n in new and old[n] != new[n])
    missing = sorted(n for n in old if n not in new)
    print(json.dumps({"old": len(old), "new": len(new), "differ": len(differ), "missing": len(missing), "added": len(set(new) - set(old)),
                      "differing": differ, "missing_names": missing}))
    return 1 if differ or missing else 0


if __name__ == "__main__":
    sys.exit(main())
