"""The option table and the option scope of tests/support.py, without a GPU: OPTION_DEFAULTS must be the library's own
initial values, and `options` must put every option it changed back where the context started."""
import os
import re

import pytest

from tests.support import HERE, OPTION_DEFAULTS, options

CSRC = os.path.join(os.path.dirname(HERE), 'advancedliteratemachinery_b200', 'csrc')


def test_option_defaults_are_the_ctx_initializers():
    """every integer option of alm_set_option is in the table, with the initializer of its field in struct Ctx"""
    with open(os.path.join(CSRC, 'c_api.cu')) as f:
        table = re.search(r'kIntOptions\[\] = \{(.*?)\n\};', f.read(), re.S).group(1)
    names = re.findall(r'\{"(\w+)", &Ctx::(\w+),', table)
    assert all(n == field for n, field in names)
    assert sorted(OPTION_DEFAULTS) == sorted(n for n, _ in names)
    with open(os.path.join(CSRC, 'alm_internal.h')) as f:
        ctx = re.search(r'\nstruct Ctx \{(.*?)\n\};', f.read(), re.S).group(1)
    for name, value in OPTION_DEFAULTS.items():
        init = re.findall(rf'(?<![\w"]){name} = (-?\d+)[,;]', ctx)
        assert init == [str(value)], name


class RecordingContext:
    """a context stub: the options' current values and every set_option call"""

    def __init__(self, **opts):
        self.opts = dict(OPTION_DEFAULTS, **opts)
        self.calls = []

    def set_option(self, key, value):
        self.calls.append((key, value))
        self.opts[key] = value


def test_options_restore_after_an_exception(monkeypatch):
    monkeypatch.delenv('ALM_OCR_OPTIONS', raising=False)
    c = RecordingContext()
    with pytest.raises(RuntimeError):
        with options(c, nsplit=1, gemm_impl=1, wattn_impl=0):
            assert (c.opts['nsplit'], c.opts['gemm_impl'], c.opts['wattn_impl']) == (1, 1, 0)
            raise RuntimeError('the body fails')
    assert c.opts == OPTION_DEFAULTS
    assert c.calls[3:] == [('nsplit', 3), ('gemm_impl', 0), ('wattn_impl', 3)]
    # ALM_OCR_OPTIONS is what a new context starts with: the scope goes back to its values, not the library's
    monkeypatch.setenv('ALM_OCR_OPTIONS', 'xattn_impl=2, wattn_impl=1,')
    c = RecordingContext(xattn_impl=2, wattn_impl=1)
    with pytest.raises(RuntimeError):
        with options(c, xattn_impl=0, wattn_impl=3, use_graphs=0):
            raise RuntimeError('the body fails')
    assert c.opts == dict(OPTION_DEFAULTS, xattn_impl=2, wattn_impl=1)
