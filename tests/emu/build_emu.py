"""Translate the CUDA sources of log_b200/csrc (kernels and the C entry points) to host C++ on top of the SIMT emulation
in tests/emu/cuda_runtime.h and build tests/emu/_build/libemu.so.  Test infrastructure only.

The translation touches exactly three constructs, mechanically:
  kernel<<<grid, block, smem, stream>>>(args);   ->  emu::launch(dim3(grid), dim3(block), smem, [=]() { kernel(args); });
  extern __shared__ T name[];                    ->  T* name = reinterpret_cast<T*>(emu::dyn_smem());
  the inline-PTX helper functions of lgr_blend.cu (PTX_HELPERS)  ->  host versions in emu_blend_helpers.h
Everything else (the kernel bodies) is compiled verbatim.
"""
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, 'log_b200', 'csrc')
BUILD = os.path.join(HERE, '_build')
LIB = os.path.join(BUILD, 'libemu.so')
SOURCES = sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))      # every kernel file and the C entry points
# inline-PTX helpers of lgr_blend.cu, replaced by tests/emu/emu_blend_helpers.h
PTX_HELPERS = ['ex2_approx', 'rcp_approx', 'smem_u32', 'lds_f4', 'lds_f2', 'sts_f32', 'pin_reg', 'red_shared_max_u32', 'red_shared_add_f32',
               'prefetch_l2', 'ldsm_x4', 'mma_tf32']


def _split_top(s):
    out, depth, cur = [], 0, ''
    for ch in s:
        if ch in '([{':
            depth += 1
        elif ch in ')]}':
            depth -= 1
        if ch == ',' and depth == 0:
            out.append(cur.strip())
            cur = ''
        else:
            cur += ch
    out.append(cur.strip())
    return out


def drop_ptx_helpers(src: str) -> str:
    """Remove the definitions of PTX_HELPERS (whole functions) and include the host versions in their place."""
    first = True
    for name in PTX_HELPERS:
        m = re.search(r'^__device__ __forceinline__ [\w ]+? ' + name + r'\(', src, flags=re.M)
        if not m:
            continue
        a = src.index('{', m.end())
        depth, b = 1, a
        while depth:
            b += 1
            depth += {'{': 1, '}': -1}.get(src[b], 0)
        repl = '}  // namespace lgr\n#include "emu_blend_helpers.h"\nnamespace lgr {\n' if first else ''
        first = False
        src = src[:m.start()] + repl + src[b + 1:]
    assert 'asm' not in re.sub(r'//.*', '', src), 'inline PTX left in the translated source'
    return src


def translate(src: str) -> str:
    src = drop_ptx_helpers(src)
    src = re.sub(r'extern\s+__shared__\s+(\w+)\s+(\w+)\[\];', r'\1* \2 = reinterpret_cast<\1*>(emu::dyn_smem());', src)
    out, pos = '', 0
    while True:
        k = src.find('<<<', pos)
        if k < 0:
            return out + src[pos:]
        # kernel name (with optional template arguments) ends right before '<<<'
        j = k
        while src[j - 1].isspace():
            j -= 1
        if src[j - 1] == '>':
            depth, j = 1, j - 1
            while depth:
                j -= 1
                depth += {'>': 1, '<': -1}.get(src[j], 0)
        while src[j - 1].isalnum() or src[j - 1] in '_:':
            j -= 1
        name = src[j:k].strip()
        e = src.index('>>>', k)
        cfg = _split_top(src[k + 3:e])
        assert 2 <= len(cfg) <= 4, cfg
        a = e + 3
        while src[a].isspace():
            a += 1
        assert src[a] == '(', src[a:a + 40]
        depth, b = 1, a
        while depth:
            b += 1
            depth += {'(': 1, ')': -1}.get(src[b], 0)
        args = src[a + 1:b]
        smem = cfg[2] if len(cfg) > 2 else '0'
        out += src[pos:j] + f'emu::launch(dim3({cfg[0]}), dim3({cfg[1]}), (size_t)({smem}), [=]() {{ {name}({args}); }})'
        pos = b + 1


def build(force=False, asan=None):
    """asan=True (or LGR_EMU_ASAN=1 in the environment): AddressSanitizer build, libemu_asan.so -- run the emulated tests
    with it as  LGR_EMU_ASAN=1 LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest
    tests/test_emulated_kernels.py tests/test_emulated_pipeline.py tests/test_emulated_host.py tests/test_tree_traverse.py
    (a CPU stand-in for compute-sanitizer memcheck: out-of-bounds accesses of global buffers and of __shared__ arrays)."""
    global LIB
    asan = bool(int(os.environ.get('LGR_EMU_ASAN', '0'))) if asan is None else asan
    tsan = int(os.environ.get('LGR_EMU_TSAN', '0'))      # ThreadSanitizer build (2: CTAs of a launch left unordered), see cuda_runtime.h
    extra = os.environ.get('LGR_EMU_EXTRA', '').split()      # e.g. -DLGR_AGG_ATOMICS=1: compile-time knobs of the kernels
    tag = ('_' + ''.join(ch for ch in ''.join(extra) if ch.isalnum())) if extra else ''
    LIB = os.path.join(BUILD, (('libemu_tsan%d' % tsan) if tsan else 'libemu_asan' if asan else 'libemu') + tag + '.so')
    os.makedirs(BUILD, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in SOURCES] + [os.path.join(CSRC, 'lgr_common.cuh'), os.path.join(CSRC, 'lgr_prof.cuh'),
                                                       os.path.join(HERE, 'cuda_runtime.h'), os.path.join(HERE, 'emu_api.cpp'), os.path.join(HERE, 'emu_blend_helpers.h'),
                                                       os.path.abspath(__file__), os.path.join(ROOT, 'include', 'log_b200_raster.h')]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    objs = []
    for f in SOURCES:
        cpp = os.path.join(BUILD, f.replace('.cu', '.emu.cpp'))
        with open(cpp, 'w') as fh:
            fh.write(f'// generated from log_b200/csrc/{f} by tests/emu/build_emu.py -- do not edit\n')
            fh.write(translate(open(os.path.join(CSRC, f)).read()))
        objs.append(cpp)
    # a 3-CTA grid for the tree walk: every emulated CTA costs 256 fibers, and 3 CTAs make the grid-stride loops iterate
    # and a counter of the tile lists that reach the LSD sort (tests/emu/cuda_runtime.h)
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fPIC', '-shared', '-w', '-DLGR_TREE_GRID=3', '-DLGR_REGION_GRID=2',
           '-DLGR_ON_LSD_FALLBACK()=emu_count_lsd_fallback()'] + extra + \
          (['-fsanitize=thread', '-DEMU_TSAN'] + (['-DEMU_TSAN_UNORDERED_CTAS'] if tsan == 2 else []) if tsan else ['-fsanitize=address', '-fno-omit-frame-pointer'] if asan else []) + ['-I', HERE, '-I', CSRC, '-o', LIB + '.tmp'] + objs + \
          [os.path.join(HERE, 'emu_api.cpp')]
    env = dict(os.environ)
    env.pop('CC', None)
    env.pop('CXX', None)
    subprocess.check_call(cmd, env=env)
    os.replace(LIB + '.tmp', LIB)
    return LIB


if __name__ == '__main__':
    print(build(force=True))
