"""Plumbing shared by the test modules: host builds of the kernel emulations, the synthetic models of the GPU tests,
the module-scoped context, scoped library options, and small helpers for guards, bits and merge results."""
import contextlib
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden')
GUARD = 1024
NAN = float('nan')


def golden(name):
    return np.load(os.path.join(GOLDEN, name))


# ----------------------------------------------------------------------------------------------- host emulations
_EMU = {}


@functools.cache
def _emu_dir():
    """One directory for every emulation library of the process, removed at interpreter exit."""
    return tempfile.TemporaryDirectory(prefix='alm_emu_')


def emu(name, bind):
    """tests/emu/<name>.cpp (kernel bodies as plain C++) built for the host once per process and loaded; `bind(lib)`
    sets the restype / argtypes of its functions.  No FMA contraction, so the host arithmetic is the device's."""
    if name not in _EMU:
        if shutil.which('g++') is None:
            pytest.skip('g++ not available')
        so = os.path.join(_emu_dir().name, name + '.so')
        subprocess.check_call(['g++', '-O1', '-ffp-contract=off', '-shared', '-fPIC', '-std=c++17',
                               os.path.join(HERE, 'emu', name + '.cpp'), '-o', so])
        lib = C.CDLL(so)
        bind(lib)
        _EMU[name] = lib
    return _EMU[name]


# ----------------------------------------------------------------------------------------------- models
_MODELS = {}


def close_models(kind=None):
    """Closes the models omni_model / mgp_model built ('omni' or 'mgp' ones only, given a kind)."""
    for k in [k for k in _MODELS if kind in (None, k[0])]:
        _MODELS.pop(k).ctx.close()


@pytest.fixture(scope='module', autouse=True)
def release_models():
    """Closes every model built for the module, so none outlives it (each holds its weights and workspace on the
    device).  Every module that uses omni_model or mgp_model imports it."""
    yield
    close_models()


def omni_model(gold, kie=False, workspace_mb=4096):
    """The OmniParserB200 of a synthetic checkpoint: seed gold['wseed'], pt_eos_bias gold['pt_eos_bias'] and, with
    `kie`, gold['vie'] entity categories.  One OmniParser is resident at a time: another checkpoint or workspace closes
    it.  gold['pt_seq_length'] / gold['rec_length'], where gold has them, are set on the vocabulary at every call."""
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from tests.conftest import omni_sd
    wseed, bias, vie = int(gold['wseed']), float(gold['pt_eos_bias']), int(gold['vie']) if kie else 0
    key = ('omni', wseed, bias, vie, workspace_mb)
    if key not in _MODELS:
        close_models('omni')
        sd = W.omniparser_state_dict(seed=wseed, vie_categories=vie, pt_eos_bias=bias) if kie else omni_sd(wseed, bias)
        _MODELS[key] = OmniParserB200(sd, OmniVocab(vie_categories=vie), workspace_mb=workspace_mb)
    m = _MODELS[key]
    for k in ('pt_seq_length', 'rec_length'):
        if k in gold:
            setattr(m.vocab, k, int(gold[k]))
    return m


def mgp_model(wseed=0):
    """The MGPSTRB200 of the synthetic MGP-STR checkpoint of seed `wseed`."""
    from advancedliteratemachinery_b200 import MGPSTRB200
    from tests.conftest import mgp_sd
    key = ('mgp', wseed)
    if key not in _MODELS:
        _MODELS[key] = MGPSTRB200(mgp_sd(wseed))
    return _MODELS[key]


# ----------------------------------------------------------------------------------------------- context and options
@pytest.fixture(scope='module')
def ctx(request):
    """One context for the module; its workspace is the module's WORKSPACE_MB where it sets one."""
    from advancedliteratemachinery_b200 import _lib
    assert torch.cuda.is_available(), 'GPU tests need an H100; there is no CPU fallback to test'
    c = _lib.Context(0)
    if hasattr(request.module, 'WORKSPACE_MB'):
        c.set_option('workspace_mb', request.module.WORKSPACE_MB)
    yield c
    c.close()


# the integer options of alm_set_option and their initial values (struct Ctx, csrc/alm_internal.h)
OPTION_DEFAULTS = dict(nsplit=3, gemm_impl=0, xattn_impl=0, fuse_ln_gemv=1, kv_decoders=3, attn_impl=0, wattn_impl=3,
                       enc_grid_cap=0, dec_grid_cap=0, xattn_ctas_per_sm=2, xattn_wg=1, sattn_wide=1, debug_skip=0,
                       decode_priority=0, small_grid_cap=0, decode_streams=2, use_graphs=1, joint_decode=1,
                       profile_gemm=0)


def initial_options():
    """The options a new context has: OPTION_DEFAULTS with ALM_OCR_OPTIONS ("name=value,...") applied over them, parsed
    as _lib.Context parses it."""
    opts = dict(OPTION_DEFAULTS)
    for kv in filter(None, os.environ.get('ALM_OCR_OPTIONS', '').split(',')):
        k, v = kv.split('=')
        opts[k.strip()] = int(v)
    return opts


@contextlib.contextmanager
def options(ctx, **kw):
    """Sets the options `kw` on `ctx` for the body; afterwards, also when the body raises, each one is back at the value
    the context was created with."""
    initial = initial_options()
    try:
        for k, v in kw.items():
            ctx.set_option(k, v)
        yield
    finally:
        for k in kw:
            ctx.set_option(k, initial[k])


# ----------------------------------------------------------------------------------------------- small helpers
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(t):
    """an fp32 tensor as its int32 bits (other tensors as they are), for bit-for-bit comparisons"""
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def guarded(n, dtype=torch.float32, fill=NAN, guard=GUARD):
    """(first n elements, whole buffer) of a device buffer with `guard` elements of `fill` after it"""
    full = torch.full((n + guard,), fill, dtype=dtype, device='cuda')
    return full[:n], full


def assert_guard(full, n, fill=NAN):
    g = full[n:]
    assert torch.equal(bits(g), bits(torch.full_like(g, fill))), 'write past the end of the output'


def assert_same(a, b):
    """Two merge results (dicts of arrays) are equal, floats bit for bit."""
    assert a.keys() == b.keys()
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.shape == y.shape and x.dtype == y.dtype, k
        if x.dtype.kind == 'f':
            u = np.uint64 if x.itemsize == 8 else np.uint32
            x, y = x.view(u), y.view(u)
        assert np.array_equal(x, y), k


def same(a, b):
    """Two spot_tiled results are equal, floats bit for bit (== on Python floats, with the keys in order)."""
    assert [[list(d.items()) for d in r] for r in a] == [[list(d.items()) for d in r] for r in b]


def kw(gold, **extra):
    """the tile layout and input sizes of a tile fixture, as spot_tiled / kie_tiled keywords"""
    return dict(tile=int(gold['tile']), overlap=int(gold['overlap']), test_min_size=int(gold['test_min_size']),
                test_max_size=int(gold['test_max_size']), **extra)
