"""Compare per-function SASS of two sm_90a binaries (objects or shared libraries) with cuobjdump -sass.

Every function of OLD must disassemble to the same SASS in NEW.  `--rename 'PATTERN=>REPLACEMENT'` (a regular expression over the
mangled name) maps a parent function to the name it has in NEW, e.g. a template parameter inserted into an existing kernel."""
import argparse, re, subprocess, sys


def functions(path):
    out = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name: funcs[name] = body
            # an anonymous namespace's mangled name carries hashes of the source path: drop them
            name, body = re.sub(r"_GLOBAL__N__[0-9a-f]+_(\d+_\w+?_cu)_[0-9a-f]+", r"_GLOBAL__N__\1", m.group(1)), []
            continue
        if name is None: continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m: body.append(re.sub(r"\s+", " ", m.group(1)))
    if name: funcs[name] = body
    return funcs


ap = argparse.ArgumentParser()
ap.add_argument("old"); ap.add_argument("new"); ap.add_argument("--rename", action="append", default=[])
a = ap.parse_args()
old, new = functions(a.old), functions(a.new)
ren = [r.split("=>", 1) for r in a.rename]
bad = 0
for name, body in sorted(old.items()):
    target = name
    for s, t in ren:
        target = re.sub(s, t, target)
    if target not in new:
        print("MISSING", name, "->", target); bad += 1
    elif new[target] != body:
        print("DIFFERS", name, len(body), len(new[target])); bad += 1
    else:
        print("same   ", name, len(body))
mapped = set()
for n in old:
    for s, t in ren:
        n = re.sub(s, t, n)
    mapped.add(n)
added = sorted(set(new) - mapped)
for n in added: print("new    ", n, len(new[n]))
print("%d of %d parent functions identical, %d new" % (len(old) - bad, len(old), len(added)))
sys.exit(1 if bad else 0)
