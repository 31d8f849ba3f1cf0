""" The ctypes mirror of PinnTerm (pinn_multi_step_terms) matches the C layout, and the caps the engine applies are the
header's (no GPU needed). """
import ctypes as C
import os
import re
import subprocess

from pydens_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'pinn_b200.h')


def test_pinn_term_layout_matches_c(tmp_path):
    src = tmp_path / 'term.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pinn_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(PinnTerm), offsetof(PinnTerm, plan),'
                   ' offsetof(PinnTerm, n_points), offsetof(PinnTerm, point_weight), offsetof(PinnTerm, points));'
                   'return 0;}\n')
    exe = tmp_path / 'term'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    T = _native.PinnTerm
    assert got == [C.sizeof(T), T.plan.offset, T.n_points.offset, T.point_weight.offset, T.points.offset]


def test_term_caps_match_the_header():
    src = open(HEADER).read()
    caps = dict(re.findall(r'#define\s+(PINN_MAX_TERM\w*)\s+(\d+)', src))
    assert int(caps['PINN_MAX_TERMS']) == _native.MAX_TERMS
    assert int(caps['PINN_MAX_TERM_POINTS']) == _native.MAX_TERM_POINTS
