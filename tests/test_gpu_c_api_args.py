"""GPU: argument handling of the C API (c_api.cu) and the entry points that share one implementation.

* every alm_set_option key: the values it accepts and the code it returns for the ones it refuses;
* a host pointer handed to an op entry point is refused with ALM_ERR_INVALID before any device work, and the context
  stays usable: alm_op_layernorm (every pointer) and alm_op_linear (bias) among them;
* alm_op_linear is alm_op_gemm with a column bias and a dense output, and alm_op_self_attention_step is
  alm_op_self_attention_step_anc with the identity ancestry: both pairs give bit-identical results.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

OK, ERR_INVALID, ERR_STATE = 0, -1, -4


@pytest.fixture
def ctx():
    from advancedliteratemachinery_b200 import _lib
    assert torch.cuda.is_available(), 'GPU tests need an H100; there is no CPU fallback to test'
    c = _lib.Context(0)
    c.set_option('workspace_mb', 1024)
    yield c
    c.close()


def _op(ctx, name, *args):
    torch.cuda.synchronize()
    return getattr(ctx.lib, name)(ctx.h, *args)


def _bits(t):
    return t.contiguous().view(torch.int32)


# ----------------------------------------------------------------------------------------------- alm_set_option
# key: (accepted values, refused values); every refusal is ALM_ERR_INVALID
SET_OPTIONS = {
    'nsplit': ([1, 3], [-1, 0, 2, 4, 5, 31, 32, 2 ** 33 + 1]),
    'gemm_impl': ([0, 1], [-1, 2, 3]),
    'xattn_impl': ([0, 1, 2], [-1, 3, 4]),
    'kv_decoders': ([1, 2, 3], [-1, 0, 4]),
    'attn_impl': ([0, 1], [-1, 2]),
    'wattn_impl': ([0, 1, 3], [-1, 2, 4, 5]),
    'xattn_ctas_per_sm': ([1, 2, 3], [-1, 0, 4]),
    'xattn_wg': ([1, 2], [-1, 0, 3]),
    'decode_streams': ([1, 2], [-1, 0, 3]),
}
FLAG_OPTIONS = ['fuse_ln_gemv', 'sattn_wide', 'decode_priority', 'use_graphs', 'profile_gemm']
ANY_OPTIONS = ['enc_grid_cap', 'dec_grid_cap', 'debug_skip', 'small_grid_cap']


def _set(ctx, key, value):
    return ctx.lib.alm_set_option(ctx.h, None if key is None else key.encode(), value)


@pytest.mark.parametrize('key', sorted(SET_OPTIONS))
def test_set_option_value_sets(ctx, key):
    accepted, refused = SET_OPTIONS[key]
    for v in refused:
        assert _set(ctx, key, v) == ERR_INVALID, (key, v)
        assert key in ctx.lib.alm_last_error(ctx.h).decode()
    for v in accepted:
        assert _set(ctx, key, v) == OK, (key, v)


def test_set_option_flags_and_free_values(ctx):
    for key in FLAG_OPTIONS:
        for v in (0, 1, 2, -1, 2 ** 40):
            assert _set(ctx, key, v) == OK, (key, v)
    for key in ANY_OPTIONS:
        for v in (0, 7, -3):
            assert _set(ctx, key, v) == OK, (key, v)
    for v in (16, 0):
        assert _set(ctx, 'trace_gemm', v) == OK


def test_set_option_unknown_keys_and_workspace(ctx):
    for key in ('nope', '', 'NSPLIT', None):
        assert _set(ctx, key, 1) == ERR_INVALID, key
    assert _set(ctx, 'workspace_mb', 63) == ERR_STATE
    assert _set(ctx, 'workspace_mb', 64) == OK
    assert _set(ctx, 'workspace_mb', 512) == OK
    A, out = torch.randn(4, 64, device='cuda'), torch.empty(4, 4, device='cuda')
    ctx.check(_op(ctx, 'alm_op_linear', A.data_ptr(), A.data_ptr(), None, out.data_ptr(), 4, 4, 64, 0, 1))
    assert _set(ctx, 'workspace_mb', 1024) == ERR_STATE   # the workspace exists now


# ----------------------------------------------------------------------------------------------- host pointers
def _layernorm_ok(ctx):
    x = torch.randn(5, 128, device='cuda')
    g, b = torch.randn(128, device='cuda'), torch.randn(128, device='cuda')
    y = torch.empty(5, 128, device='cuda')
    ctx.check(_op(ctx, 'alm_op_layernorm', x.data_ptr(), g.data_ptr(), b.data_ptr(), 1e-5, y.data_ptr(), 5, 128))
    ref = torch.nn.functional.layer_norm(x.double(), (128,), g.double(), b.double(), 1e-5)
    assert float((y.double() - ref).abs().max()) < 1e-4


@pytest.mark.parametrize('host', ['x', 'gamma', 'beta', 'y'])
def test_layernorm_refuses_host_pointers(ctx, host):
    bufs = {'x': torch.randn(5, 128), 'gamma': torch.ones(128), 'beta': torch.zeros(128), 'y': torch.zeros(5, 128)}
    dev = {k: (v if k == host else v.cuda()) for k, v in bufs.items()}
    rc = _op(ctx, 'alm_op_layernorm', dev['x'].data_ptr(), dev['gamma'].data_ptr(), dev['beta'].data_ptr(), 1e-5,
             dev['y'].data_ptr(), 5, 128)
    assert rc == ERR_INVALID
    assert 'alm_op_layernorm' in ctx.lib.alm_last_error(ctx.h).decode()
    assert torch.equal(bufs['y'], torch.zeros(5, 128))
    _layernorm_ok(ctx)


def test_linear_refuses_host_bias(ctx):
    M, N, K = 8, 16, 32
    A, W = torch.randn(M, K, device='cuda'), torch.randn(N, K, device='cuda')
    out = torch.zeros(M, N, device='cuda')
    bias = torch.randn(N)
    assert _op(ctx, 'alm_op_linear', A.data_ptr(), W.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K, 0, 1) == ERR_INVALID
    assert 'alm_op_linear' in ctx.lib.alm_last_error(ctx.h).decode()
    bd = bias.cuda()
    ctx.check(_op(ctx, 'alm_op_linear', A.data_ptr(), W.data_ptr(), bd.data_ptr(), out.data_ptr(), M, N, K, 0, 1))
    ref = A.double() @ W.double().T + bd.double()
    assert float((out.double() - ref).abs().max()) < 1e-4


def _d(*shape, dt=torch.float32):
    return torch.zeros(*shape, dtype=dt, device='cuda')


def _h(*shape, dt=torch.float32):
    return torch.zeros(*shape, dtype=dt)


def _planes(hi, out, keep):
    from advancedliteratemachinery_b200 import _lib
    a = _lib.GemmOperand(hi.data_ptr(), None, 8, 16, 16, 1, 1, 0, 0)
    e = _lib.GemmEpilogue()
    e.out_f32, e.ldo, e.obs0, e.alpha = out.data_ptr(), 8, 64, 1.0
    keep += [hi, out, a, e]
    return C.byref(a), C.byref(a), C.byref(e)


def _page(keep):
    img = _d(32, 32, 3, dt=torch.uint8)
    rgb, hw = (C.c_void_p * 1)(img.data_ptr()), (C.c_int * 1)(32)
    quad, pi = (C.c_float * 8)(2, 2, 20, 2, 20, 10, 2, 10), (C.c_int * 1)(0)
    keep += [img, rgb, hw, quad, pi]
    return rgb, hw, hw, 1, quad, pi


def _cfg(keep):
    from advancedliteratemachinery_b200 import _lib
    cfg = _lib.DecodeCfg()
    keep.append(cfg)
    return C.byref(cfg)


def _p(keep, t):
    keep.append(t)
    return t.data_ptr()


# one host pointer at each entry point: (entry point, arguments after the context), built from `keep`-bound helpers
REFUSALS = {
    'gemm_A': lambda k, p: ('alm_op_gemm', p(_h(8, 16)), p(_d(8, 16)), 8, 8, 16, 1, 1, p(_d(64)), None, None, 8, 64,
                            None, 0, 0, 1.0, 0, None, 0, 0, None, None, 0, 0),
    'gemm_out': lambda k, p: ('alm_op_gemm', p(_d(8, 16)), p(_d(8, 16)), 8, 8, 16, 1, 1, p(_h(64)), None, None, 8, 64,
                              None, 0, 0, 1.0, 0, None, 0, 0, None, None, 0, 0),
    'gemm_planes_hi': lambda k, p: ('alm_op_gemm_planes', *_planes(_h(8, 16, dt=torch.bfloat16), _d(64), k)),
    'gemm_planes_out': lambda k, p: ('alm_op_gemm_planes', *_planes(_d(8, 16, dt=torch.bfloat16), _h(64), k)),
    'linear_A': lambda k, p: ('alm_op_linear', p(_h(8, 16)), p(_d(8, 16)), None, p(_d(64)), 8, 8, 16, 0, 1),
    'attention': lambda k, p: ('alm_op_attention', p(_d(4, 192)), p(_h(4, 64)), 1, 4, 1),
    'gemv': lambda k, p: ('alm_op_gemv', p(_h(16)), None, 0, p(_d(8, 16)), None, None, p(_d(8)), 1, 8, 16, 0, None,
                          None, None, 0),
    'self_attention_step': lambda k, p: ('alm_op_self_attention_step', p(_h(1, 1536)), p(_d(1, 4, 512)),
                                         p(_d(1, 4, 512)), p(_d(1, 512)), 1, 0, 4),
    'self_attention_step_anc': lambda k, p: ('alm_op_self_attention_step_anc', p(_d(1, 1536)), p(_d(1, 4, 512)),
                                             p(_d(1, 4, 512)), p(_d(1, 512)), 1, 0, 4, p(_h(1, 4, dt=torch.int32))),
    'cross_attention': lambda k, p: ('alm_op_cross_attention', p(_h(1, 512)), p(_d(8, 512)), p(_d(8, 512)), None,
                                     p(_d(1, 512)), 1, 0, 1, 1, 8, 0, 0, 1),
    'rec_locations': lambda k, p: ('alm_op_rec_locations', p(_d(1, 512)), p(_h(8, 512)), None, None,
                                   p(_h(1, dt=torch.int32) + 4), p(_d(1, 8)), 1, 1, 8, 0),
    'head_select': lambda k, p: ('alm_op_head_select', p(_h(1, 8)), 1, 8, 8, 0, 0, _cfg(k), p(_d(1, dt=torch.int32)),
                                 p(_d(1)), None, None),
    'beam_select': lambda k, p: ('alm_op_beam_select', p(_d(2, 8)), 1, 2, 8, 8, 0, _cfg(k), p(_h(2)),
                                 p(_d(2, dt=torch.int32)), p(_d(2, dt=torch.int32)), p(_d(2, dt=torch.int32)), p(_d(2))),
    'pre_quad_crops': lambda k, p: ('alm_pre_quad_crops', *_page(k), 1, 32, 128, p(_h(3, 32, 128))),
}


@pytest.mark.parametrize('case', sorted(REFUSALS))
def test_op_refuses_a_host_pointer(ctx, case):
    keep = []
    name, *args = REFUSALS[case](keep, lambda t: _p(keep, t))
    assert _op(ctx, name, *args) == ERR_INVALID
    _layernorm_ok(ctx)


# ----------------------------------------------------------------------------------------------- shared implementations
@pytest.mark.parametrize('nsplit', [3, 1])
@pytest.mark.parametrize('M,N,K,batch,act,with_bias', [(37, 70, 44, 3, 1, True), (64, 96, 64, 1, 0, False),
                                                        (5, 24, 20, 2, 2, True)])
def test_linear_is_gemm_with_a_column_bias(ctx, nsplit, M, N, K, batch, act, with_bias):
    ctx.set_option('nsplit', nsplit)
    g = torch.Generator(device='cuda').manual_seed(M * N + K)
    A = torch.randn(batch, M, K, generator=g, device='cuda')
    W = torch.randn(batch, N, K, generator=g, device='cuda')
    bias = torch.randn(batch, N, generator=g, device='cuda')[0].contiguous() if with_bias else None
    bp = bias.data_ptr() if with_bias else None
    lin = torch.full((batch, M, N), float('nan'), device='cuda')
    gem = torch.full((batch, M, N), float('nan'), device='cuda')
    ctx.check(_op(ctx, 'alm_op_linear', A.data_ptr(), W.data_ptr(), bp, lin.data_ptr(), M, N, K, act, batch))
    ctx.check(_op(ctx, 'alm_op_gemm', A.data_ptr(), W.data_ptr(), M, N, K, batch, batch, gem.data_ptr(), None, None, N,
                  M * N, bp, 1 if with_bias else 0, 0, 1.0, act, None, 0, 0, None, None, 0, 0))
    assert torch.isfinite(lin).all()
    assert torch.equal(_bits(lin), _bits(gem))


@pytest.mark.parametrize('wide', [1, 0])
def test_self_attention_step_is_anc_with_identity(ctx, wide):
    ctx.set_option('sattn_wide', wide)
    S, t, Tmax = 12, 5, 16
    g = torch.Generator(device='cuda').manual_seed(wide)
    qkv = torch.randn(S, 1536, generator=g, device='cuda')
    kc0 = torch.randn(S, Tmax, 512, generator=g, device='cuda')
    vc0 = torch.randn(S, Tmax, 512, generator=g, device='cuda')
    anc = torch.arange(S, dtype=torch.int32, device='cuda')[:, None].expand(S, Tmax).contiguous()
    res = []
    for name, extra in (('alm_op_self_attention_step', ()), ('alm_op_self_attention_step_anc', (anc.data_ptr(),))):
        kc, vc, out = kc0.clone(), vc0.clone(), torch.full((S, 512), float('nan'), device='cuda')
        ctx.check(_op(ctx, name, qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(), S, t, Tmax, *extra))
        res.append((out, kc, vc))
    assert torch.isfinite(res[0][0]).all()
    for a, b in zip(*res):
        assert torch.equal(_bits(a), _bits(b))
