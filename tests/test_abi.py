# -*- coding: utf-8 -*-
"""CPU checks of the drop-in boundary: libpia_b200.so loads without a GPU and exports every symbol
include/pia_b200.h declares, with a ctypes signature for each (no compute calls here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    from painlessinferenceacceleration_b200.build import build_library
    so = build_library()
    return ctypes.CDLL(so)


def _declared():
    hdr = open(os.path.join(ROOT, 'include', 'pia_b200.h')).read()
    hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
    return sorted(set(re.findall(r'\b(pia_[a-z0-9_]+)\s*\(', hdr)))


def test_every_declared_symbol_is_exported(lib):
    names = _declared()
    assert len(names) >= 25
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_ctypes_table_matches_header():
    from painlessinferenceacceleration_b200 import _lib
    assert sorted(_lib.SYMBOLS) == _declared()
    L = _lib.load()
    assert L.pia_abi_version() == 3  # v3: pia_rmsnorm / pia_rmsnorm_partials take the rounding of x_hat
    # (v2: request slots (pia_slots_t), device-resident max_length / idx)
    assert L.pia_launch_count() == 0
    assert L.pia_last_error() is not None


def test_header_cites_the_reference_for_every_entry_point():
    hdr = open(os.path.join(ROOT, 'include', 'pia_b200.h')).read()
    # each functional block names the reference file:line it replaces
    for anchor in ('lookahead_cache.py:349-373', 'lookahead_cache.py:375-406', 'lookahead_cache.py:408-439',
                   ':243-308', 'pretrained_model.py:764-892', 'pretrained_model.py:863-875'):
        assert anchor in hdr, anchor


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'painlessinferenceacceleration_b200')
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                src = open(os.path.join(d, f)).read()
                assert 'import oracle' not in src and 'from oracle' not in src, os.path.join(d, f)
                cited = src.replace('/root/reference/lookahead/lookahead', '<ref>').replace('/root/reference/flood/flood', '<ref>')
                assert '/root/reference' not in cited or f.endswith('.py')   # citations in comments only


def test_no_cpu_fallback_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    with pytest.raises(RuntimeError):
        LookaheadCache()


def test_ctypes_struct_layouts_match_the_header(tmp_path):
    """sizeof / field offsets of every struct that crosses the ABI by pointer, measured by compiling the header with gcc"""
    import subprocess
    from painlessinferenceacceleration_b200 import _lib
    src = tmp_path / 'layout.c'
    structs = {'pia_trie_config_t': _lib.TrieConfig, 'pia_trie_stats_t': _lib.TrieStats,
               'pia_attn_config_t': _lib.AttnConfig, 'pia_accept_config_t': _lib.AcceptConfig,
               'pia_slots_t': _lib.Slots}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/pia_b200.h"', 'int main(void){']
    for cname, cls in structs.items():
        lines.append(f'printf("{cname} %zu", sizeof({cname}));')
        for fname, _t in cls._fields_:
            lines.append(f'printf(" %zu", offsetof({cname}, {fname}));')
        lines.append('printf("\\n");')
    lines += ['return 0;}']
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = subprocess.check_output([str(exe)]).decode().strip().split('\n')
    for line, (cname, cls) in zip(out, structs.items()):
        parts = line.split()
        assert parts[0] == cname
        assert int(parts[1]) == ctypes.sizeof(cls), cname
        assert [int(x) for x in parts[2:]] == [getattr(cls, f).offset for f, _ in cls._fields_], cname
