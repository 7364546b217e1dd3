"""Compare the kernel SASS of two builds of libtidbgpu.so, function by function, with addresses stripped.

    python tools/sass_diff.py OLD.so NEW.so

A kernel defined in a header that several sources include appears once per object file; its copies are compared as a
sorted list.  Prints the functions only one build has and the functions whose instructions differ; exits 1 if any differ."""
import re
import subprocess
import sys


def functions(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs, body = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            body = []
            funcs.setdefault(m.group(1), []).append(body)
        elif body is not None and "/*" in line:
            ins = re.sub(r"/\*[0-9a-f]{4,}\*/|/\* 0x[0-9a-f]+ \*/", "", line).strip()
            if ins:
                body.append(ins)
    return {n: sorted(bodies) for n, bodies in funcs.items()}


def main(old_lib, new_lib):
    old, new = functions(old_lib), functions(new_lib)
    count = lambda f: sum(len(b) for b in f.values())
    print(f"{count(old)} functions in {old_lib}, {count(new)} in {new_lib}")
    for n in sorted(old.keys() - new.keys()):
        print("only in old:", n)
    for n in sorted(new.keys() - old.keys()):
        print("only in new:", n)
    changed = sorted(n for n in old.keys() & new.keys() if old[n] != new[n])
    for n in changed:
        print("differs:", n)
    print(f"{len(old.keys() & new.keys()) - len(changed)} common functions identical, {len(changed)} differ")
    return 1 if changed else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1], sys.argv[2]))
