"""What the upstream watsor code returned in the comparison tests, stored so the comparisons run without a checkout.

`upstream(module, key, compute)` returns the upstream side of a comparison: with an upstream checkout present it calls
`compute()` (which imports and runs the upstream code) and checks the result against the stored value; without one it
returns the stored value from tests/golden/reference/<module>.json.  WATSOR_RECORD_GOLDEN=1 (with a checkout) rewrites
the stored values instead of checking them.  Values are JSON: lists, dicts, strings, numbers."""
import json
import os

import pytest

from oracle.reference_build import has_reference

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference')
RECORD = os.environ.get('WATSOR_RECORD_GOLDEN') == '1'
_cache = {}


def _path(module):
    return os.path.join(GOLDEN, module + '.json')


def _load(module):
    if module not in _cache:
        p = _path(module)
        _cache[module] = json.load(open(p)) if os.path.isfile(p) else {}
    return _cache[module]


def _plain(v):
    return json.loads(json.dumps(v))


def upstream(module, key, compute):
    data = _load(module)
    if has_reference():
        value = _plain(compute())
        if RECORD:
            data[key] = value
            os.makedirs(GOLDEN, exist_ok=True)
            with open(_path(module), 'w') as f:
                json.dump(data, f, sort_keys=True, separators=(',', ':'))
        else:
            assert key in data, 'no stored upstream value for %s / %s (record with WATSOR_RECORD_GOLDEN=1)' % (module, key)
            assert data[key] == value, 'upstream output differs from the stored one: %s / %s' % (module, key)
        return value
    if key not in data:
        pytest.skip('no stored upstream value for %s / %s' % (module, key))
    return data[key]
