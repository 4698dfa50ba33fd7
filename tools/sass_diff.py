"""Device-code regression check without a GPU: do the kernels of two libvlpk.so builds have identical SASS?

    git archive <validated-commit> vlp_b200/csrc include | tar -x -C /tmp/val && make -C /tmp/val/vlp_b200/csrc -j8
    python tools/sass_diff.py /tmp/val/vlp_b200/libvlpk.so vlp_b200/libvlpk.so

Shows whether a host-side change left every kernel of an already validated build byte-identical."""
import hashlib
import re
import subprocess
import sys


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    ks, cur, buf = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if cur:
                ks[cur] = hashlib.md5("\n".join(buf).encode()).hexdigest()
            cur, buf = m.group(1), []
        elif cur and "/*" in line:
            # instruction text without addresses / encodings; cuobjdump pads every line to the widest instruction of the whole
            # dump, so the padding changes with any kernel and is collapsed
            buf.append(" ".join(re.sub(r"/\*[^*]*\*/", " ", line).split()))
    if cur:
        ks[cur] = hashlib.md5("\n".join(buf).encode()).hexdigest()
    # anonymous-namespace prefixes carry a per-file hash
    return {re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_(\w+?)_cu_[0-9a-f]+", r"ANON_\1", k): v for k, v in ks.items()}


def main(old, new):
    a, b = kernels(old), kernels(new)
    diff = sorted(k for k in a if k in b and a[k] != b[k])
    gone = sorted(k for k in a if k not in b)
    added = sorted(k for k in b if k not in a)
    print(f"{len(a)} kernels in {old}; {len(b)} in {new}: identical {len(a) - len(diff) - len(gone)}, changed {len(diff)}, "
          f"removed {len(gone)}, new {len(added)}")
    for tag, names in (("changed", diff), ("removed", gone), ("new", added)):
        for k in names:
            print(f"  {tag}: {k[:150]}")
    return 1 if diff or gone else 0


if __name__ == "__main__":
    try:
        sys.exit(main(sys.argv[1], sys.argv[2]))
    except BrokenPipeError:
        sys.exit(0)
