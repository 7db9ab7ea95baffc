"""The programmatic-dependent-launch (PDL) window rule of the fused engine, shared by tests/test_launch_order_cpu.py (launch
plans recorded on the CPU) and tests/test_gpu_launch_order.py (launches recorded on the device).

A kernel launched with the PDL attribute may start as soon as the kernel before it in the stream has executed
``griddepcontrol.launch_dependents``; until its own ``griddepcontrol.wait`` it runs beside that kernel, and beside every
kernel that one was itself running beside.  What it reads before the wait must therefore not be written by any launch of
that window:

    window(B) = the launches before B, walking back, while each triggers its dependents early; the walk includes a
                triggering launch and goes on past it only if that launch itself has the PDL attribute.

A launch that does not trigger early (every ``<<<>>>`` kernel of the library, a torch kernel, a copy, a host synchronise)
closes the window.  Launches torch issues between library calls are not seen here, so the check treats every window as if
they were absent: it can only be stricter than the device.

``PREWAIT`` names, per kernel, what it reads before its wait.  The kernels carry the same list in a comment next to their
``griddepcontrol.wait`` (``// PDL pre-wait reads: ...``), and the CPU test checks the two against each other."""
import ctypes
import os
import re
import struct

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'openscene_b200', 'csrc')

# kernel -> operands read before griddepcontrol.wait (names resolved to address ranges per entry point in launch_of)
PREWAIT = {
    'k_conv_tc': ('nbr', 'scale', 'shift'),
    'k_conv_finish': (),
    'k_conv_chain': (),
}
# entry point -> the PDL kernels it launches (all of them trigger at their first instruction when launched with PDL)
PDL_ENTRY = {
    'osb_conv_fwd_tc': ('k_conv_tc', 'k_conv_finish'),
    'osb_convtr_fwd_tc': ('k_conv_tc',),
    'osb_conv_chain_launch': ('k_conv_chain',),
}
# entry points that launch nothing (host-side planners and queries): invisible to the stream
HOST_ONLY = {'osb_version', 'osb_last_error', 'osb_device_info', 'osb_launch_count', 'osb_conv_desc_fill', 'osb_conv_desc_bytes',
             'osb_conv_chain_grid', 'osb_tuning_set'}

_DESC_FMT = '<12Q q 14i 8i'
_DESC_PTRS = ('src0', 'src1', 'nbr', 'wtiles', 'scale', 'shift', 'res', 'out_split', 'out_f32', 'out_row_map', 'cmap', 'partial')
_DESC_INTS = ('K', 'nb0', 'nb1', 'cout', 'cout_pad', 'nt', 'n_ntiles', 'relu', 'cmap_cout', 'nsplit', 'm_tiles', 'nsub_max',
              'barrier_before', 'stages_per_split')
DESC_BYTES = struct.calcsize(_DESC_FMT)


def is_host_only(name):
    return name in HOST_ONLY or name.endswith('_bytes')


def ival(a):
    """ctypes argument -> int (pointers) / float"""
    if a is None:
        return 0
    if isinstance(a, (int, float)):
        return a
    return a.value or 0


def decode_descs(descs_host, n_layers):
    raw = ctypes.string_at(descs_host, DESC_BYTES * n_layers)
    out = []
    for i in range(n_layers):
        v = struct.unpack(_DESC_FMT, raw[DESC_BYTES * i:DESC_BYTES * (i + 1)])
        d = dict(zip(_DESC_PTRS, v[:12]))
        d['n_out'] = v[12]
        d.update(zip(_DESC_INTS, v[13:27]))
        out.append(d)
    return out


class Launch:
    """One library entry point as the stream sees it: PDL attribute, early trigger, operands by name, writes."""
    __slots__ = ('name', 'pdl', 'triggers', 'operands', 'writes')

    def __init__(self, name, pdl, operands=None, writes=()):
        self.name, self.pdl, self.triggers = name, bool(pdl), bool(pdl)
        self.operands = operands or {}                 # name -> [(lo, hi)]
        self.writes = list(writes)                     # [(lo, hi, label)]

    def prewait(self, table=None):
        table = PREWAIT if table is None else table
        out = []
        for k in PDL_ENTRY.get(self.name, ()):
            for op in table[k]:
                out += [(lo, hi, f'{k}.{op}') for (lo, hi) in self.operands.get(op, ())]
        return out


def _rng(p, nbytes):
    return [(p, p + nbytes)] if p and nbytes > 0 else []


def launch_of(name, args):
    """Launch of a recorded entry point (``args`` as passed to the library; chain launches decode their host descriptors).
    None for host-only entry points."""
    if is_host_only(name):
        return None
    if name not in PDL_ENTRY:
        return Launch(name, False)                     # every other entry point: <<<>>> launches, copies, host syncs
    a = [ival(x) for x in args]
    if name == 'osb_conv_fwd_tc':
        (s0, c0, _, s1, c1, _, nbr, n_out, K, _, cout, scale, shift, res, _, osp, of, _, ws, ws_b, flags, _) = a
        ops = {'nbr': _rng(nbr, 4 * K * n_out), 'scale': _rng(scale, 4 * cout), 'shift': _rng(shift, 4 * cout)}
        w = [(lo, hi, 'out_split') for lo, hi in _rng(osp, 4 * n_out * cout)]
        w += [(lo, hi, 'out_f32') for lo, hi in _rng(of, 4 * n_out * cout)]
        w += [(lo, hi, 'split workspace') for lo, hi in _rng(ws, ws_b)]
        return Launch(name, flags & 1, ops, w)
    if name == 'osb_convtr_fwd_tc':
        (src, cin, n_c, cmap, kvol, _, cout, scale, shift, _, osp, of, flags, _) = a
        ops = {'scale': _rng(scale, 4 * cout), 'shift': _rng(shift, 4 * cout), 'nbr': []}
        w = [(lo, hi, 'out_split') for lo, hi in _rng(osp, 4 * kvol * n_c * cout)]
        w += [(lo, hi, 'out_f32') for lo, hi in _rng(of, 4 * kvol * n_c * cout)]
        return Launch(name, flags & 1, ops, w)
    if name == 'osb_conv_chain_launch':
        descs, n_layers, gbar, flags, _ = a
        layers = decode_descs(descs, n_layers)
        ops = {'gbar': _rng(gbar + 4, 4) if gbar else []}
        w = [(lo, hi, 'grid barrier') for lo, hi in _rng(gbar, 16)]
        for li, d in enumerate(layers):
            rows = 8 * d['n_out'] if d['cmap'] else d['n_out']
            oc = d['cmap_cout'] if d['cmap'] else d['cout']
            w += [(lo, hi, f'layer {li} out_split') for lo, hi in _rng(d['out_split'], 4 * rows * oc)]
            w += [(lo, hi, f'layer {li} out_f32') for lo, hi in _rng(d['out_f32'], 4 * rows * oc)]
            if d['nsplit'] > 1:
                w += [(lo, hi, f'layer {li} partials') for lo, hi in _rng(d['partial'], 4 * d['nsplit'] * d['n_out'] * d['cout_pad'])]
    return Launch(name, flags & 1, ops, w)


def check_windows(seq, table=None):
    """seq: [Launch] in stream order.  Returns (windows checked, launches in them, violations)."""
    seq = [L for L in seq if L is not None]
    bad, n_win, n_in = [], 0, 0
    for i, B in enumerate(seq):
        if not B.pdl:
            continue
        reads = B.prewait(table)
        win, j = [], i - 1
        while j >= 0 and seq[j].triggers:
            win.append((j, seq[j]))
            if not seq[j].pdl:
                break
            j -= 1
        n_win += 1
        n_in += len(win)
        for j, P in win:
            for (wlo, whi, wl) in P.writes:
                for (rlo, rhi, rl) in reads:
                    if wlo < rhi and rlo < whi:
                        bad.append(f"launch {i} ({B.name}) reads {rl} before its griddepcontrol.wait, and launch {j} "
                                   f"({P.name}) of its PDL window writes it ({wl})")
    return n_win, n_in, bad


def source_prewait():
    """{kernel: operands} from the ``// PDL pre-wait reads: ...`` comments next to every griddepcontrol.wait in csrc/, and
    the set of kernels that trigger their dependents early"""
    marks, triggers = {}, set()
    for fn in sorted(os.listdir(CSRC)):
        if not fn.endswith(('.cu', '.cuh')):
            continue
        lines = open(os.path.join(CSRC, fn)).read().split('\n')
        kernel = None
        for i, ln in enumerate(lines):
            m = re.search(r'__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(', ln)
            if m is None and i > 0 and re.search(r'__global__', lines[i - 1]):
                m = re.search(r'^\s*(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(', ln)
            if m:
                kernel = m.group(1)
            if 'griddepcontrol.launch_dependents' in ln:
                triggers.add(kernel)
            if 'griddepcontrol.wait' in ln and not ln.strip().startswith('//'):
                mk = re.search(r'PDL pre-wait reads:\s*(.*)$', lines[i - 1])
                assert mk, f"{fn}:{i + 1}: griddepcontrol.wait in {kernel} without a '// PDL pre-wait reads:' comment above it"
                ops = re.sub(r'\(.*\)', '', mk.group(1)).strip()          # a parenthesised remark is not an operand
                names = () if ops == 'none' else tuple(re.match(r'\s*(\w+)', x).group(1) for x in ops.split(','))
                assert kernel not in marks, f"{kernel}: two griddepcontrol.wait"
                marks[kernel] = names
    return marks, triggers
