"""Compare the SASS of two builds of libctt_b200_msm.so function by function.
Usage: python tools/sass_diff.py old.so new.so

Runs `cuobjdump -sass` on both files and splits each listing at its `Function :` headers. Functions are matched by name, so a
different order of functions in the cubins is not a change; a name that occurs in several cubins (a `static` kernel compiled
into several translation units) is compared as the sorted list of its bodies. Offsets and branch / call targets in a listing
are relative to the function's own section, so identical code gives identical text, up to whitespace: cuobjdump pads the
columns of a whole cubin to its widest instruction, so a change in one function re-pads its neighbours, and runs of whitespace
are collapsed before comparing. Prints the functions added, removed and changed; exits with 1 on any difference."""
import subprocess
import sys
from collections import defaultdict


def functions(path):
    """name -> sorted list of instruction texts, one per cubin that defines the function"""
    out = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    bodies = defaultdict(list)
    name, body = None, []

    def flush():
        if name is not None:
            bodies[name].append("\n".join(body))

    for line in out.splitlines():
        s = line.strip()
        if s.startswith("Function :"):
            flush()
            name, body = s[len("Function :"):].strip(), []
        elif s.startswith("Fatbin "):        # the next cubin's header: not part of the last function
            flush()
            name, body = None, []
        elif name is not None:
            body.append(" ".join(line.split()))
    flush()
    return {k: sorted(v) for k, v in bodies.items()}


def main():
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    removed = sorted(old.keys() - new.keys())
    added = sorted(new.keys() - old.keys())
    changed = sorted(k for k in old.keys() & new.keys() if old[k] != new[k])
    for title, names in (("removed", removed), ("added", added), ("changed", changed)):
        for k in names:
            print("%s: %s" % (title, k))
    print("%d functions compared: %d removed, %d added, %d changed" % (len(old.keys() | new.keys()), len(removed), len(added), len(changed)))
    sys.exit(1 if removed or added or changed else 0)


if __name__ == "__main__":
    main()
