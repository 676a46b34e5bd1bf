#!/usr/bin/env python3
"""Symbolic tracer for straight-line fp32 SASS (sm_90).

Purpose: derive the exact FMA association the reference kernels were compiled to (nvcc fuses in
NVVM *and* again in ptxas, so neither the C source nor the PTX is authoritative) so that the
oracle (fmaf) and our kernels (__fmaf_rn) can pin the same association and produce bit-identical
depth keys / radii / tile rectangles.  See DESIGN.md "bit-exact binning".

Walks one function linearly (branches are not taken; predicated non-branch ops are skipped and
reported), keeps a hash-consed expression DAG per register, and prints a let-style listing of
every value that reaches a store or a float compare.  IEEE division / rcp / sqrt expansions are
folded back into DIV / RCP / SQRT nodes.

usage: sass_trace.py file.sass <function-substring> [--params name:size,name:size,...]
"""
import re
import sys

PARAMS = {}
UNIQ = '--uniq' in sys.argv
if UNIQ: sys.argv.remove('--uniq')
LEAFY = ('leaf', 'const', 'ptr', 'ptrhi')


def pname(off):
    return PARAMS.get(off, f'c[{hex(off)}]')


class DAG:
    def __init__(self):
        self.nodes = []
        self.index = {}

    def mk(self, op, *args):
        key = (op,) + args
        if key in self.index:
            return self.index[key]
        self.nodes.append(key)
        self.index[key] = len(self.nodes) - 1
        return len(self.nodes) - 1

    def leaf(self, name):
        return self.mk('leaf', name)

    def const(self, v):
        return self.mk('const', v)


def parse_operand(tok):
    tok = tok.strip().replace('.reuse', '')
    neg = ab = False
    if tok.startswith('-'):
        neg, tok = True, tok[1:]
    if tok.startswith('|') and tok.endswith('|'):
        ab, tok = True, tok[1:-1]
    return neg, ab, tok


def trace(lines):
    g = DAG()
    regs = {}
    ctr = [0]
    out = []

    def val(tok):
        neg, ab, t = parse_operand(tok)
        if t == 'RZ' or t == 'URZ':
            n = g.const('0')
        elif re.fullmatch(r'U?R\d+', t):
            n = regs[t] if t in regs else g.leaf('undef_' + t)
        elif t.startswith('c['):
            cm = re.search(r'c\[0x0\]\[(0x[0-9a-f]+)\]', t)
            n = g.leaf(pname(int(cm.group(1), 16)) if cm else t)
        else:
            n = g.const(t)
        if ab:
            n = g.mk('abs', n)
        if neg:
            n = g.mk('neg', n)
        return n

    def isptr(t):
        t = t.replace('.reuse', '')
        return t in regs and g.nodes[regs[t]][0] in ('ptr', 'ptrhi')

    # pre-pass: instruction list with addresses, to decide which predicated forward branches
    # guard a slow-path CALL (IEEE div/rcp/sqrt fix-up) and must be treated as taken.
    ins = []
    for ln in lines:
        m = re.search(r'/\*([0-9a-f]{4,5})\*/\s+(.*?);', ln)
        if m:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    skip_until = -1
    for ia, (iaddr, txt) in enumerate(ins):
        if iaddr < skip_until:
            continue
        addr = f'{iaddr:04x}'
        bm = re.match(r'@!?U?P\w+\s+BRA(?:\.U)?\s+(?:!?U?P\w+,\s*)?(0x[0-9a-f]+)', txt)
        if bm:
            tgt = int(bm.group(1), 16)
            if tgt > iaddr and any(a2 < tgt and a2 > iaddr and t2.split()[0].startswith('CALL')
                                   for a2, t2 in ins[ia:ia + 40]):
                skip_until = tgt
                continue
        pred = None
        pm = re.match(r'(@!?U?P\w+)\s+(.*)', txt)
        if pm:
            pred, txt = pm.group(1), pm.group(2)
        parts = txt.split(None, 1)
        op = parts[0]
        args = [a.strip() for a in parts[1].split(',')] if len(parts) > 1 else []
        base = op.split('.')[0]
        if pred and base not in ('BRA', 'EXIT'):
            if base in ('FFMA', 'FMUL', 'FADD', 'MUFU', 'FSEL', 'MOV'):
                out.append(f'   [skipped predicated {addr}: {pred} {txt}]')
            continue
        if not args:
            continue
        dst = args[0].replace('.reuse', '')
        mreg = re.fullmatch(r'(U?R)(\d+)', dst)

        def sib(k):
            return f'{mreg.group(1)}{int(mreg.group(2)) + k}'

        if base in ('LDC', 'LDCU') and mreg:
            cm = re.search(r'c\[0x0\]\[(0x[0-9a-f]+)\]', args[-1])
            if cm:
                off = int(cm.group(1), 16)
                if '.64' in op and (off + 4) in PARAMS and not PARAMS[off + 4].endswith('.hi'):
                    regs[dst] = g.leaf(pname(off))
                    regs[sib(1)] = g.leaf(pname(off + 4))
                elif '.64' in op:
                    regs[dst] = g.mk('ptr', pname(off))
                    regs[sib(1)] = g.mk('ptrhi', pname(off))
                else:
                    regs[dst] = g.leaf(pname(off))
            else:
                regs[dst] = g.leaf(f'{base}@{addr}')
            continue
        if base in ('IMAD', 'LEA', 'IADD3', 'IADD', 'UIADD3', 'UIMAD', 'ULEA', 'MOV', 'UMOV') and mreg \
                and any(isptr(a) for a in args[1:]):
            pn = [regs[a.replace('.reuse', '')] for a in args[1:] if isptr(a)][-1]
            kind, nm = g.nodes[pn][0], g.nodes[pn][1]
            if base in ('MOV', 'UMOV'):
                regs[dst] = pn
            elif '.HI' in op or kind == 'ptrhi':
                regs[dst] = g.mk('ptrhi', nm)
            else:
                nm2 = nm if nm.endswith('+i') else nm + '+i'
                regs[dst] = g.mk('ptr', nm2)
                if '.WIDE' in op:
                    regs[sib(1)] = g.mk('ptrhi', nm2)
            continue
        if base in ('LDG', 'LD', 'LDS') and mreg:
            src = args[-1]
            width = 4 if '.128' in op else 2 if '.64' in op else 1
            am = re.search(r'\[(U?R\d+)(?:\.64)?(?:\+(-?0x[0-9a-f]+))?\]$', src)
            name = None
            if am and am.group(1) in regs and g.nodes[regs[am.group(1)]][0] == 'ptr':
                name = f'{g.nodes[regs[am.group(1)]][1]}[{int(am.group(2) or "0x0", 16) // 4}]'
            for k in range(width):
                ctr[0] += 1
                nm = name if name else f'ld{ctr[0]}@{addr}'
                if width > 1 and name:
                    base_i = int(am.group(2) or "0x0", 16) // 4 + k
                    nm = f'{g.nodes[regs[am.group(1)]][1]}[{base_i}]'
                regs[sib(k)] = g.leaf(nm + (f'#{addr}' if '+i' in nm and UNIQ else ''))
            continue
        if base == 'FFMA':
            regs[dst] = g.mk('fma', val(args[1]), val(args[2]), val(args[3]))
        elif base == 'FMUL':
            regs[dst] = g.mk('mul', val(args[1]), val(args[2]))
        elif base == 'FADD':
            regs[dst] = g.mk('add', val(args[1]), val(args[2]))
        elif base == 'FMNMX':
            kind = 'max' if args[3].strip() == '!PT' else 'min'
            regs[dst] = g.mk(kind, val(args[1]), val(args[2]))
        elif base == 'MUFU':
            regs[dst] = g.mk(op.split('.')[1].lower(), val(args[1]))
        elif base == 'MOV' or base == 'UMOV':
            regs[dst] = val(args[1])
        elif base in ('FRND', 'F2F', 'F2I', 'I2F', 'I2FP', 'F2FP'):
            regs[dst] = g.mk(op.lower(), val(args[-1]))
            if '.F64' in op.split('.')[1:2] or op.startswith('F2F.F64') or op.startswith('I2F.F64'):
                regs[sib(1)] = g.leaf('hi')
        elif base in ('DADD', 'DMUL', 'DFMA'):
            regs[dst] = g.mk(base.lower(), *[val(a) for a in args[1:]])
        elif base == 'FSEL':
            regs[dst] = g.mk('fsel', val(args[1]), val(args[2]), g.leaf(args[3]))
        elif base in ('STG', 'ST', 'STS'):
            am = re.search(r'\[(U?R\d+)(?:\.64)?(?:\+(-?0x[0-9a-f]+))?\]$', args[0])
            where = args[0]
            if am and am.group(1) in regs and g.nodes[regs[am.group(1)]][0] == 'ptr':
                where = f'{g.nodes[regs[am.group(1)]][1]}[{int(am.group(2) or "0x0", 16) // 4}]'
            sreg = args[1].replace('.reuse', '')
            width = 4 if '.128' in op else 2 if '.64' in op else 1
            sm = re.fullmatch(r'(U?R)(\d+)', sreg)
            for k in range(width):
                r = f'{sm.group(1)}{int(sm.group(2)) + k}' if sm else sreg
                out.append((addr, f'STORE {where}+{k}', r, regs.get(r)))
        elif base == 'FSETP':
            out.append((addr, f'{op} a', args[2], val(args[2])))
            out.append((addr, f'{op} b', args[3], val(args[3])))
        elif mreg:
            regs[dst] = g.leaf(f'{base}@{addr}')
    return g, out


def matchers(g):
    N = g.nodes

    def is_(n, op):
        return N[n][0] == op

    def rcp_refined(n):
        if not is_(n, 'fma'):
            return None
        a, b, c = N[n][1:]
        if a != c or not is_(a, 'rcp'):
            return None
        den = N[a][1]
        if is_(b, 'fma'):
            x, y, z = N[b][1:]
            if is_(x, 'neg') and N[x][1] == den and y == a and is_(z, 'const'):
                return den
            if is_(y, 'neg') and N[y][1] == den and x == a and is_(z, 'const'):
                return den
            if is_(y, 'add') and x == a:   # fma(r0, add(-den,-0), 1)
                p = N[y][1]
                if is_(p, 'neg') and N[p][1] == den:
                    return den
        if is_(b, 'add'):
            p, q = N[b][1:]
            if is_(p, 'neg') and is_(N[p][1], 'fma'):
                x, y, z = N[N[p][1]][1:]
                if x == den and y == a:
                    return den
        return None

    def div(n):
        if not is_(n, 'fma'):
            return None
        r1, rem, q = N[n][1:]
        den = rcp_refined(r1)
        if den is None or not is_(q, 'fma') or not is_(rem, 'fma'):
            return None
        qa, qb, qc = N[q][1:]
        if qb != r1:
            return None
        ra, rb, rc = N[rem][1:]
        den_ok = (is_(ra, 'neg') and N[ra][1] == den) or \
                 (is_(ra, 'add') and is_(N[ra][1], 'neg') and N[N[ra][1]][1] == den)
        if den_ok and rb == q and rc == qa:
            return (qa, den)
        return None

    def sqrt(n):
        if not is_(n, 'fma'):
            return None
        e, h, s = N[n][1:]
        if not (is_(s, 'mul') and is_(h, 'mul') and is_(e, 'fma')):
            return None
        x, r = N[s][1:]
        if is_(r, 'rsq') and N[r][1] == x:
            return x
        if is_(x, 'rsq') and N[x][1] == r:
            return r
        return None

    return rcp_refined, div, sqrt


def dagprint(g, out):
    N = g.nodes
    rcp_refined, div, sqrt = matchers(g)
    names = {}
    lines = []

    def ref(n):
        if n is None:
            return '?'
        k = N[n]
        if k[0] in LEAFY:
            return str(k[1])
        if k[0] == 'neg':
            return '-' + ref(k[1])
        if k[0] == 'abs':
            return '|' + ref(k[1]) + '|'
        if n in names:
            return names[n]
        d = div(n)
        if d:
            body = f'DIV({ref(d[0])}, {ref(d[1])})'
        else:
            r = rcp_refined(n)
            if r is not None:
                body = f'RCP({ref(r)})'
            else:
                q = sqrt(n)
                if q is not None:
                    body = f'SQRT({ref(q)})'
                else:
                    body = f'{k[0]}(' + ', '.join(ref(a) for a in k[1:]) + ')'
        nm = f't{len(names)}'
        names[n] = nm
        lines.append(f'  {nm} = {body}')
        return nm

    for o in out:
        if isinstance(o, str):
            lines.append(o)
            continue
        addr, what, reg, n = o
        lines.append(f'{addr} {what} <- {reg} = {ref(n)}')
    print('\n'.join(lines))


def main():
    if '--params' in sys.argv:
        i = sys.argv.index('--params')
        spec = sys.argv[i + 1]
        del sys.argv[i:i + 2]
        off = 0x380
        for item in spec.split(','):
            nm, sz = item.split(':')
            sz = int(sz)
            al = min(sz, 8)
            off = (off + al - 1) // al * al
            if sz in (4, 8):
                PARAMS[off] = nm
                if sz == 8:
                    PARAMS[off + 4] = nm + '.hi'
            else:
                for k in range(0, sz, 4):
                    PARAMS[off + k] = f'{nm}.{k // 4}'
            off += sz
    path, fn = sys.argv[1], sys.argv[2]
    lines = open(path).read().split('\n')
    start = None
    end = len(lines)
    for i, l in enumerate(lines):
        if 'Function :' in l:
            if start is not None:
                end = i
                break
            if fn in l:
                start = i
    g, out = trace(lines[start:end])
    dagprint(g, out)


main()
