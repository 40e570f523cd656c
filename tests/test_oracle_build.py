"""oracle/Makefile: after the build nothing is out of date, and a changed header recompiles exactly the objects whose
sources include it, directly or through another header, and relinks libsm_oracle.so.  No GPU; the header checks are
make's dry runs, so they write nothing."""
import glob
import os
import re
import subprocess

import pytest

import oracle_lib as O

DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")


def _includes(path):
    """the quoted includes of `path`, followed through the headers, as make names them (relative to oracle/)"""
    found, todo = set(), [path]
    while todo:
        cur = todo.pop()
        with open(cur) as f:
            text = f.read()
        for name in re.findall(r'^\s*#\s*include\s+"([^"]+)"', text, re.M):
            inc = os.path.normpath(os.path.join(os.path.dirname(cur), name))
            if inc not in found:
                found.add(inc)
                todo.append(inc)
    return {os.path.relpath(p, DIR) for p in found}


INCLUDES = {os.path.basename(src)[:-3] + ".o": _includes(src) for src in glob.glob(os.path.join(DIR, "*.cc"))}


def test_nothing_is_out_of_date_after_the_build():
    O.build()
    r = subprocess.run(["make", "-C", DIR, "-q"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("header", sorted(set().union(*INCLUDES.values())))
def test_a_changed_header_rebuilds_exactly_its_includers(header):
    O.build()
    r = subprocess.run(["make", "-C", DIR, "-n", "-W", header], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    compiled = set(re.findall(r" -c -o (\S+\.o) ", r.stdout))
    assert compiled == {obj for obj, inc in INCLUDES.items() if header in inc}, r.stdout
    assert " -shared -o libsm_oracle.so " in r.stdout, r.stdout
