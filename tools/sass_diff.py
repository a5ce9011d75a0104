#!/usr/bin/env python
"""Compare the machine code of two builds function by function:
    python tools/sass_diff.py old/libeld_b200.so new/libeld_b200.so     # or two `cuobjdump -sass` dumps
Prints each function whose SASS differs, and whether only the register numbers, only the control words (stalls,
barriers, reuse) or the instructions themselves differ.  Given two .so files it also prints each function whose
`cuobjdump -res-usage` line (registers, shared memory, stack, ...) differs.  Exits 1 on any difference."""
import os
import re
import subprocess
import sys

CUOBJDUMP = os.environ.get('CUOBJDUMP', '/usr/local/cuda/bin/cuobjdump')
INSN = re.compile(r'\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;\s*/\* (0x[0-9a-f]+) \*/')
WORD = re.compile(r'\s*/\* (0x[0-9a-f]+) \*/\s*$')
REG = re.compile(r'\bU?R\d+\b|\bU?P\d\b')


def sass(path):
    """{function: [[instruction, encoding], ...]}"""
    text = subprocess.run([CUOBJDUMP, '-sass', path], check=True, capture_output=True, text=True).stdout \
        if path.endswith('.so') else open(path).read()
    out, cur = {}, None
    for line in text.splitlines():
        if m := re.match(r'\s*Function : (\S+)', line):
            out[m.group(1)] = cur = []
        elif cur is not None and (m := INSN.match(line)):
            cur.append([m.group(1), m.group(2)])
        elif cur and (m := WORD.match(line)):
            cur[-1][1] += m.group(1)
    return out


def res_usage(path):
    text = subprocess.run([CUOBJDUMP, '-res-usage', path], check=True, capture_output=True, text=True).stdout
    return dict(re.findall(r'Function (\S+):\n\s*(.*)', text))


def demangle(name):
    try:
        return subprocess.run(['c++filt', name], capture_output=True, text=True).stdout.strip() or name
    except OSError:
        return name


def main(old, new):
    a, b = sass(old), sass(new)
    diffs = 0
    for name in sorted(set(a) | set(b)):
        if name not in a or name not in b:
            kind = 'only in ' + (old if name in a else new)
        elif a[name] == b[name]:
            continue
        elif [i for i, _ in a[name]] == [i for i, _ in b[name]]:
            kind = 'control words only'
        elif [REG.sub('R', i) for i, _ in a[name]] == [REG.sub('R', i) for i, _ in b[name]]:
            kind = 'register numbers only'
        else:
            kind = 'instructions (%d -> %d)' % (len(a[name]), len(b[name]))
        diffs += 1
        print('SASS   %-26s %s' % (kind, demangle(name)))
    if old.endswith('.so') and new.endswith('.so'):
        ra, rb = res_usage(old), res_usage(new)
        for name in sorted(set(ra) | set(rb)):
            if ra.get(name) != rb.get(name):
                diffs += 1
                print('USAGE  %s\n    %s\n -> %s' % (demangle(name), ra.get(name), rb.get(name)))
    print('%d difference(s) over %d functions' % (diffs, len(set(a) | set(b))))
    return 1 if diffs else 0


if __name__ == '__main__':
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
