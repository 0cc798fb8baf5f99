"""Turn a traced plant graph (symtrace.py) into C / CUDA source.

Output = two text blobs:
  * tables:  `PLANT_TABLE(name, n) = {...};` for every breakpoint / value / slope array that survives
  * body:    straight-line SSA statements computing xdot[] from X[] and U[]

Passes: dead-code elimination from the live derivative outputs; lookup specialisation (a 2-D lookup whose
first argument is a constant collapses to a 1-D lookup over a pre-blended column; slope tables are
pre-divided in double with the reference's operation order so results stay bit-identical); sharing of
the breakpoint search between lookups on the same (axis, input); in the double-precision device build, long searches
become certified bucketed searches (bucket.py).
"""
import math

import bucket
import symtrace as S


def hexf(x):
    if x != x:
        return '(0.0/0.0)'
    if x in (float('inf'), float('-inf')):
        return '(1.0/0.0)' if x > 0 else '(-1.0/0.0)'
    return float(x).hex()


def tables_text(tabs):
    out = []
    for name in sorted(tabs):
        vals = tabs[name]
        out.append('PLANT_TABLE(%s, %d) = {' % (name, len(vals)))
        for i in range(0, len(vals), 4):
            out.append('  ' + ', '.join(hexf(x) for x in vals[i:i + 4]) + ',')
        out.append('};')
    return '\n'.join(out)


class ConstPool:
    """double literals that do not fit a 32-bit immediate (low word != 0) are pooled into one array (`PLANT_K(i)`): on the
    device that array lives in constant memory, so DFMA/DMUL/DSETP take them as c[bank][offset] operands instead of
    materialising every 64-bit literal with two uniform-register moves."""

    def __init__(self):
        self.index = {}
        self.vals = []

    def ref(self, x):
        import struct
        bits = struct.unpack('<Q', struct.pack('<d', x))[0]
        if (bits & 0xffffffff) == 0 or x != x:
            return hexf(x)
        if bits not in self.index:
            self.index[bits] = len(self.vals)
            self.vals.append(x)
        return 'PLANT_K(%d)' % self.index[bits]

    def text(self):
        out = ['PLANT_CONSTS(%d) = {' % max(len(self.vals), 1)]
        vals = self.vals or [0.0]
        for i in range(0, len(vals), 4):
            out.append('  ' + ', '.join(hexf(x) for x in vals[i:i + 4]) + ',')
        out.append('};')
        return '\n'.join(out)


class Emitter:
    def __init__(self, tracer, real='real', pool=None, fast=False, bucket=False):
        # fast (device build only): divisions by table spacings become multiplications by pre-inverted tables and
        # sin/cos of the same angle are computed by one sincos; results move by <= 1 ulp per affected operation
        self.fast = fast
        # bucket (double-precision device build only): long breakpoint searches become certified O(1) bucketed searches
        # (bucket.py); the index is the counted one bit for bit
        self.bucket = bucket
        self.pool = pool
        self.tr = tracer
        self.tabs = {}        # name -> list of floats
        self.bkts = {}        # name -> bucket bytes of a bucketed search (bucket.py)
        self.tabname = {}     # key -> name
        self.lines = []
        self.real = real
        self.idx = {}         # (axis name, node id) -> (ivar, dvar)
        self.stats = {}

    # ---- tables ----
    @staticmethod
    def _hname(prefix, vals):
        import hashlib, struct
        h = hashlib.md5(struct.pack('<%dd' % len(vals), *vals)).hexdigest()[:10]
        return '%s%d_%s' % (prefix, len(vals), h)

    def table(self, key, prefix='T'):
        if key not in self.tabname:
            vals = list(self.tr.tables[key])
            name = self._hname(prefix, vals)
            self.tabname[key] = name
            self.tabs[name] = vals
        return self.tabname[key]

    def derived(self, tag, vals):
        key = ('derived', tuple(vals), tag)
        if key not in self.tabname:
            name = self._hname('D', list(vals))
            self.tabname[key] = name
            self.tabs[name] = list(vals)
        return self.tabname[key]

    # ---- helpers ----
    def lit(self, x):
        return self.pool.ref(x) if self.pool is not None else hexf(x)

    def ref(self, a):
        if S.is_sym(a):
            if a.op == 'const':
                return self.lit(S.fval(a.args[0]))
            return 'v%d' % a.id
        return self.lit(S.fval(a))

    def index_of(self, axis_key, unode):
        axis = self.table(axis_key)
        n = len(self.tabs[axis])
        k = (axis, unode.id)
        if k not in self.idx:
            iv = 'i%d' % len(self.idx)
            dv = 'd%d' % len(self.idx)
            # rt_GetLookupIndex (@0xf470) as a branch-free count of interior breakpoints below the input:
            # idx = #{1 <= j <= n-2 : x[j] < u}, with the reference's tie rule (u >= 0: x[i] < u <= x[i+1];
            # u < 0: x[i] <= u < x[i+1]) folded per breakpoint: a negative breakpoint compares with <=.
            xs = self.tabs[axis]
            terms = ['(%s %s %s)' % (self.lit(xs[j]), '<=' if xs[j] < 0 else '<', self.ref(unode)) for j in range(1, n - 1)]
            counted = ' + '.join(terms) if terms else '0'
            plan = bucket.plan(xs) if self.bucket else None
            if plan is not None:
                # the same index from one uniform cell: its byte (PLANT_BKT) is the count at the cell's left end and
                # the cell holds at most the one breakpoint xs[n0 + 1]; negative breakpoints' `<=` becomes `<` against
                # the next double above a negative input.  PLANT_SEARCH(bucketed, counted): the includer picks one
                # (the bucketed form needs the byte tables next to the staged tables)
                bk = plan.name()
                self.bkts[bk] = list(plan.bkt)
                y = ('plant_tie_up(%s)' if plan.tie else '%s') % self.ref(unode)
                self.lines.append('const int %s = PLANT_SEARCH(plant_bucket(%s, %s, %s, %d, PLANT_BKT(%s), PLANT_TAB(%s)), %s);'
                                  % (iv, y, self.lit(plan.s), self.lit(plan.o), plan.nb, bk, axis, counted))
            else:
                self.lines.append('const int %s = %s;' % (iv, counted))
            self.lines.append('const %s %s = %s - PLANT_TAB(%s)[%s];' % (self.real, dv, self.ref(unode), axis, iv))
            self.idx[k] = (iv, dv)
        return self.idx[k]

    def emit(self, outputs, out_names):
        live = set()
        stack = [o for o in outputs if S.is_sym(o)]
        while stack:
            n = stack.pop()
            if n.id in live:
                continue
            live.add(n.id)
            for a in n.args:
                if S.is_sym(a) and a.id not in live:
                    stack.append(a)
        R = self.real
        L = self.lines
        li = S.Tracer.lookup_index
        cnt = {}
        partner = {(n.op, n.args[0].id): n.id for n in S.G.nodes if n.id in live and n.op in ('sin', 'cos')}
        done_pair = set()
        # guards: expensive node -> (cond node id, side) when every use funnels into selects on one condition
        users = {}
        outs = {o.id for o in outputs if S.is_sym(o)}
        for n in S.G.nodes:
            if n.id in live:
                for x in n.args:
                    if S.is_sym(x):
                        users.setdefault(x.id, []).append(n)
        guards = {}
        for n in S.G.nodes:
            if n.id in live and n.op in ('exp', 'pow') and self.fast:
                conds, frontier, seen, ok = set(), [n], set(), True
                while frontier and ok:
                    m = frontier.pop()
                    if m.id in seen:
                        continue
                    seen.add(m.id)
                    if m.id in outs:
                        ok = False
                    for u in users.get(m.id, []):
                        if u.op == 'select' and m is not u.args[0]:
                            if u.args[0].op not in ('cmp', 'cmpmask'):
                                ok = False
                            conds.add((u.args[0].id, 1 if m is u.args[1] else 2))
                        elif u.op in ('add', 'sub', 'mul', 'div', 'neg'):
                            frontier.append(u)
                        else:
                            ok = False
                guards[n.id] = next(iter(conds)) if ok and len(conds) == 1 else None
        for n in S.G.nodes:
            if n.id not in live or n.op == 'const':
                continue
            cnt[n.op] = cnt.get(n.op, 0) + 1
            a = n.args
            v = 'v%d' % n.id
            op = n.op
            r = self.ref
            if op == 'X':
                L.append('const %s %s = X[%d];' % (R, v, a[0]))
            elif op == 'U':
                L.append('const %s %s = U[%d];' % (R, v, a[0]))
            elif op == 'div' and self.fast and a[1].op == 'const' and S.fval(a[1].args[0]) != 0.0:
                L.append('const %s %s = %s * %s;' % (R, v, r(a[0]), self.lit(1.0 / S.fval(a[1].args[0]))))   # x / c -> x * (1/c)
            elif op == 'div' and self.fast:
                L.append('const %s %s = PLANT_DIV(%s, %s);' % (R, v, r(a[0]), r(a[1])))
            elif op == 'sub' and a[0].op == 'const' and S.fval(a[0].args[0]) == 0.0 and math.copysign(1.0, S.fval(a[0].args[0])) < 0:
                L.append('const %s %s = -%s;' % (R, v, r(a[1])))       # -0.0 - x: a negation (one build negates by subtraction ...
            elif op == 'mul' and any(x.op == 'const' and S.fval(x.args[0]) == -1.0 for x in a[:2]):
                other = a[1] if (a[0].op == 'const' and S.fval(a[0].args[0]) == -1.0) else a[0]
                L.append('const %s %s = -%s;' % (R, v, r(other)))      # ... another by a gain of -1): the same bits either way
            elif op in ('add', 'sub', 'mul', 'div'):
                sym = {'add': '+', 'sub': '-', 'mul': '*', 'div': '/'}[op]
                L.append('const %s %s = %s %s %s;' % (R, v, r(a[0]), sym, r(a[1])))
            elif op == 'sqrt':
                L.append('const %s %s = PLANT_SQRT(%s);' % (R, v, r(a[0])))
            elif op == 'max':
                L.append('const %s %s = (%s > %s) ? %s : %s;' % (R, v, r(a[0]), r(a[1]), r(a[0]), r(a[1])))
            elif op == 'min':
                L.append('const %s %s = (%s < %s) ? %s : %s;' % (R, v, r(a[0]), r(a[1]), r(a[0]), r(a[1])))
            elif op == 'neg':
                L.append('const %s %s = -%s;' % (R, v, r(a[0])))
            elif op == 'abs':
                L.append('const %s %s = PLANT_FABS(%s);' % (R, v, r(a[0])))
            elif op in ('cmp', 'cmpmask'):
                sym = {'gt': '>', 'ge': '>=', 'lt': '<', 'le': '<=', 'eq': '==', 'ne': '!='}[a[0]]
                L.append('const bool %s = %s %s %s;' % (v, r(a[1]), sym, r(a[2])))
            elif op == 'select':
                L.append('const %s %s = %s ? %s : %s;' % (R, v, r(a[0]), r(a[1]), r(a[2])))
            elif op == 'mand':
                L.append('const %s %s = %s ? %s : 0.0;' % (R, v, r(a[0]), r(a[1])))
            elif op == 'mandn':
                L.append('const %s %s = %s ? 0.0 : %s;' % (R, v, r(a[0]), r(a[1])))
            elif op in ('sin', 'cos') and self.fast and (('cos' if op == 'sin' else 'sin'), a[0].id) in partner:
                other = partner[('cos' if op == 'sin' else 'sin'), a[0].id]
                if (op, a[0].id) not in done_pair:
                    sn, cn = (v, 'v%d' % other) if op == 'sin' else ('v%d' % other, v)
                    L.append('%s %s, %s; PLANT_SINCOS(%s, &%s, &%s);' % (R, sn, cn, r(a[0]), sn, cn))
                    done_pair.add((op, a[0].id)); done_pair.add((('cos' if op == 'sin' else 'sin'), a[0].id))
            elif op == 'tan' and self.fast and ('sin', a[0].id) in partner and ('cos', a[0].id) in partner:
                L.append('const %s %s = PLANT_DIV(v%d, v%d);' % (R, v, partner['sin', a[0].id], partner['cos', a[0].id]))
            elif op in ('exp', 'pow') and self.fast and guards.get(n.id) is not None:
                # only one side of a select consumes this value: evaluate it under that condition (both sides of the
                # ISA-atmosphere switch are otherwise computed at every stage)
                cid, side = guards[n.id]
                call = 'PLANT_EXP(%s)' % r(a[0]) if op == 'exp' else 'PLANT_POW(%s, %s)' % (r(a[0]), r(a[1]))
                L.append('%s %s = 0.0; if (%sv%d) %s = %s;' % (R, v, '' if side == 1 else '!', cid, v, call))
            elif op in ('sin', 'cos', 'tan', 'exp', 'log10', 'atan', 'asin', 'acos'):
                L.append('const %s %s = PLANT_%s(%s);' % (R, v, op.upper(), r(a[0])))
            elif op == 'pow':
                L.append('const %s %s = PLANT_POW(%s, %s);' % (R, v, r(a[0]), r(a[1])))
            elif op == 'powsnf':
                if a[1].op == 'const' and S.fval(a[1].args[0]) == 2.0:
                    L.append('const %s %s = %s * %s;' % (R, v, r(a[0]), r(a[0])))     # rt_powd_snf(x, 2) == x*x
                else:
                    L.append('const %s %s = plant_powd_snf(%s, %s);' % (R, v, r(a[0]), r(a[1])))
            elif op == 'lookup1':
                kx, ky, u = a
                xs, ys = self.tr.tables[kx], self.tr.tables[ky]
                iv, dv = self.index_of(kx, u)
                sl = [(ys[i + 1] - ys[i]) / (xs[i + 1] - xs[i]) for i in range(len(xs) - 1)]
                sn = self.derived('sl', sl)
                yn = self.table(ky)
                L.append('const %s %s = PLANT_TAB(%s)[%s] * %s + PLANT_TAB(%s)[%s];' % (R, v, sn, iv, dv, yn, iv))
            elif op == 'lookup2':
                kx, ky, kz, x, y = a
                xs, ys, zs = self.tr.tables[kx], self.tr.tables[ky], self.tr.tables[kz]
                nx, ny = len(xs), len(ys)
                if x.op == 'const':
                    xv = S.fval(x.args[0])
                    ix = li(xs, xv)
                    dx = xs[ix + 1] - xs[ix]
                    ux = xv - xs[ix]
                    col = [(zs[ix + 1 + nx * j] - zs[ix + nx * j]) / dx * ux + zs[ix + nx * j] for j in range(ny)]
                    sa = [(col[j + 1] - col[j]) / (ys[j + 1] - ys[j]) for j in range(ny - 1)]
                    an = self.derived('col', col)
                    sn = self.derived('sa', sa)
                    iv, dv = self.index_of(ky, y)
                    L.append('const %s %s = PLANT_TAB(%s)[%s] * %s + PLANT_TAB(%s)[%s];' % (R, v, sn, iv, dv, an, iv))
                    cnt['lookup2->1'] = cnt.get('lookup2->1', 0) + 1
                else:
                    sx = []
                    for j in range(ny):
                        for i in range(nx):
                            sx.append((zs[i + 1 + nx * j] - zs[i + nx * j]) / (xs[i + 1] - xs[i]) if i < nx - 1 else 0.0)
                    dy = [ys[j + 1] - ys[j] for j in range(ny - 1)]
                    sxn = self.derived('sx', sx)
                    dyn = self.derived('dy', dy)
                    zn = self.table(kz)
                    ixv, dxv = self.index_of(kx, x)
                    if y.op == 'const':
                        raise NotImplementedError('lookup2 with constant y')
                    iyv, dyv = self.index_of(ky, y)
                    L.append('const int k%d = %s + %d * %s;' % (n.id, ixv, nx, iyv))
                    L.append('const %s a%d = PLANT_TAB(%s)[k%d] * %s + PLANT_TAB(%s)[k%d];' % (R, n.id, sxn, n.id, dxv, zn, n.id))
                    L.append('const %s b%d = PLANT_TAB(%s)[k%d + %d] * %s + PLANT_TAB(%s)[k%d + %d];' % (R, n.id, sxn, n.id, nx, dxv, zn, n.id, nx))
                    if self.fast:
                        rdyn = self.derived('rdy', [1.0 / d for d in dy])
                        L.append('const %s %s = (b%d - a%d) * PLANT_TAB(%s)[%s] * %s + a%d;' % (R, v, n.id, n.id, rdyn, iyv, dyv, n.id))
                    else:
                        L.append('const %s %s = (b%d - a%d) / PLANT_TAB(%s)[%s] * %s + a%d;' % (R, v, n.id, n.id, dyn, iyv, dyv, n.id))
            elif op == 'table3':
                k1, k2, k3, k4, u0, u1, u2 = a
                t = [self.table(k) for k in (k1, k2, k3, k4)]
                ns = [len(self.tabs[x]) for x in t[:3]]
                L.append('const %s %s = plant_table3(PLANT_TAB(%s), %d, PLANT_TAB(%s), %d, PLANT_TAB(%s), %d, PLANT_TAB(%s), %s, %s, %s);'
                         % (R, v, t[0], ns[0], t[1], ns[1], t[2], ns[2], t[3], r(u0), r(u1), r(u2)))
            else:
                raise NotImplementedError(op)
        for o, name in zip(outputs, out_names):
            L.append('%s = %s;' % (name, self.ref(o)))
        self.stats = cnt
        return cnt

    def used_tables(self):
        body = '\n'.join(self.lines)
        return {name: vals for name, vals in self.tabs.items() if ('(%s)' % name) in body}

    def tables_text(self):
        used = self.used_tables()
        self.table_bytes = sum(8 * len(v) for v in used.values())
        return tables_text(used)

    def body_text(self):
        return '\n'.join(self.lines)
