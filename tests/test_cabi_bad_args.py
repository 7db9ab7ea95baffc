"""Error behaviour at the C ABI (SURVEY.md 8b: "returns int status with a thread-local error string; no exception -- and no
signal -- crosses the ABI").  Every entry point is called with all-NULL / all-zero and with negative arguments, in a child
process so that a crash would show up as a failed test instead of taking pytest down.  No GPU is needed: argument
validation happens on the host before the first CUDA call."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHILD = r'''
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
from ctypes import c_char_p, c_double, c_void_p
L = C.lib()
out = {}
for name, (res, argt) in sorted(C.SIGNATURES.items()):
    for mode in ("null", "neg"):
        args = []
        for t in argt:
            if t is c_void_p or t is c_char_p or (isinstance(t, type) and issubclass(t, ctypes._Pointer)):
                args.append(None)
            elif t is c_double:
                args.append(0.0)
            else:
                args.append(0 if mode == "null" else -1)
        r = getattr(L, name)(*args)
        err = L.osb_last_error()
        out[name + ":" + mode] = [int(r) if isinstance(r, int) else None, (err or b"").decode(errors="replace")]
print("RESULT " + json.dumps(out))
'''

# not compute entry points: constants, counters, size queries (any value is legal; they must only survive the call)
_QUERIES = {'osb_version', 'osb_last_error', 'osb_launch_count', 'osb_conv_chain_grid', 'osb_conv_desc_bytes', 'osb_device_info'}


def test_degenerate_arguments_fail_with_a_message_and_never_crash():
    p = subprocess.run([sys.executable, '-c', _CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, f"the library crashed on degenerate arguments (exit {p.returncode}):\n{p.stderr[-2000:]}"
    line = [l for l in p.stdout.splitlines() if l.startswith('RESULT ')][-1]
    res = json.loads(line[len('RESULT '):])
    from openscene_b200 import _cabi as C
    assert len(res) == 2 * len(C.SIGNATURES)
    for key, (rc, err) in res.items():
        name, mode = key.split(':')
        if name in _QUERIES or name.endswith('_bytes'):
            continue
        if name == 'osb_gather_rows_f32' and mode == 'null':
            assert rc == 0                                   # zero rows: a documented no-op
            continue
        assert rc != 0, f"{key}: accepted degenerate arguments"
        assert err.strip(), f"{key}: failed without a message"
    # size queries of rejected shapes reserve nothing
    for name in ('osb_conv_chain_workspace_bytes', 'osb_conv_tc_workspace_bytes', 'osb_conv_wgrad_tc_workspace_bytes',
                 'osb_conv_packed_weight_bytes', 'osb_conv_weight_tiles_bytes', 'osb_occgrid_bytes'):
        assert res[name + ':null'][0] == 0 and res[name + ':neg'][0] == 0, name


_K_CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
L = C.lib()
out = {}
def run(name, *args):
    return [getattr(L, name)(*args), (L.osb_last_error() or b'').decode()]
for k in (0, -1, 481, 512, 100000):
    # valid widths and counts, NULL buffers: only the text count is wrong, and it must be refused before any launch
    out['osb_match_scores:%d' % k] = run('osb_match_scores', None, 0, 10, 768, None, 10, None, k, 0, None, None, None, None)
    out['osb_match_ensemble:%d' % k] = run('osb_match_ensemble', None, None, 10, 512, None, 10, None, None, None, k, None,
                                           None, None, None)
    out['osb_match_vote:%d' % k] = run('osb_match_vote', None, 0, 10, 768, None, 10, None, k, 0, None, None, None, None,
                                       None)
print('RESULT ' + json.dumps(out))
'''


def test_match_entry_points_refuse_text_counts_outside_1_to_480_on_both_routes():
    """the tensor-core kernel streams at most five 96-row passes; both routes refuse any other K on the host"""
    for simt in ('0', '1'):
        p = subprocess.run([sys.executable, '-c', _K_CHILD, ROOT], capture_output=True, text=True, timeout=300,
                           env=dict(os.environ, OSB_MATCH_SIMT=simt))
        assert p.returncode == 0, p.stderr[-2000:]
        res = json.loads([l for l in p.stdout.splitlines() if l.startswith('RESULT ')][-1][len('RESULT '):])
        assert len(res) == 15
        for key, (rc, err) in res.items():
            assert rc != 0 and 'K_text' in err and 'outside 1..480' in err, (simt, key, rc, err)


_CONV_CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
L = C.lib()
out = {}
def run(name, *args):
    return [getattr(L, name)(*args), (L.osb_last_error() or b'').decode()]
# valid shapes (n_out 10, cin 3, cout 32, K 1 over the identity map); only the named argument is wrong.  NULL buffers
# throughout, so nothing could be launched even if a refusal were missing.
out['fwd:ld_in<cin'] = run('osb_conv_fwd_f32', None, 2, None, 10, 1, None, 3, 32, 0, None, None)
out['fwd:NULL buffers'] = run('osb_conv_fwd_f32', None, 3, None, 10, 1, None, 3, 32, 0, None, None)
out['fwd:identity map, K 27'] = run('osb_conv_fwd_f32', None, 3, None, 10, 27, None, 3, 32, 0, None, None)
out['wgrad:identity map, K 27'] = run('osb_conv_wgrad_f32', None, None, 10, 27, None, 3, 32, None, None)
out['wgrad:NULL buffers'] = run('osb_conv_wgrad_f32', None, None, 10, 1, None, 3, 32, None, None)
print('RESULT ' + json.dumps(out))
'''


def test_fp32_convolutions_refuse_bad_buffers_and_maps_with_valid_shapes():
    """osb_conv_fwd_f32 / osb_conv_wgrad_f32 refuse, on the host and before the weight gradient's memset, a row stride
    below cin, NULL operand buffers and an identity map with K != 1; each message names its cause"""
    p = subprocess.run([sys.executable, '-c', _CONV_CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith('RESULT ')][-1][len('RESULT '):])
    want = {'fwd:ld_in<cin': 'ld_in 2 < cin 3', 'fwd:NULL buffers': 'NULL buffer',
            'fwd:identity map, K 27': 'identity map requires K == 1', 'wgrad:identity map, K 27': 'identity map requires K == 1',
            'wgrad:NULL buffers': 'NULL buffer'}
    assert set(res) == set(want)
    for key, (rc, err) in res.items():
        assert rc != 0 and want[key] in err, (key, rc, err)
