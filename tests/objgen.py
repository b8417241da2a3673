"""Seeded histories of documents with many objects: maps, lists, texts and tables nested in each other, written by several
replicas at once, as binary changes (columnar.encode_change_raw).

Replicas write in rounds. Every writer of a round sees the document as it was at the start of the round: its deps are the
heads then and its startOp is the greatest op counter then plus 1, so concurrent changes share counters and actor order
breaks the ties. A small model tracks what a frontend would know: the type of each object, the live opIds of each map key
and list element (the preds of the next op there), and every element ever inserted into each list, deleted ones included,
so that later ops can name them. An `inc` leaves its counter live and is not itself live.

One change mixes ops on several objects: make* at map keys and as inserted list elements, ops into objects made earlier in
the same change, set / del / update-with-pred in maps, tables and list elements, insert runs of 1-8 elements (sometimes
alternating between two texts), counters and `inc`, `set` then `make*` on one key. Forced rounds add the shapes random
choice meets too rarely: one key overwritten concurrently by objects and scalars, 3+ actors making objects on one key at
the same counter with edits inside each afterwards (also once the key was overwritten or deleted), list / map nesting
up to `depth` levels, and tables of row maps.

`boundary=True` opens the history with list objects of exactly 2 047 / 2 048 / 2 049 / 4 095 / 4 096 / 4 097 rows and
tiny objects between them: object starts fall on both sides of the engine's scan (2 048) and radix (4 096) tiles, and
one batch holds many tiny list partitions next to several above 2 048 items.
"""
import random

from automerge_classic_b200 import columnar

TYPES = {'makeMap': 'map', 'makeList': 'list', 'makeText': 'text', 'makeTable': 'table'}
HOT_KEYS = ('a', 'b', 'c', 'ключ', 'x🐦')
BOUNDARY_ROWS = (2047, 2048, 2049, 4095, 4096, 4097)


class Model:
    """What every replica knows once it has seen a set of changes. A writer works on a View of it."""

    def __init__(self):
        self.types = {'_root': 'map'}
        self.objs = ['_root']                 # every object ever made, in creation order
        self.live = {}                        # (obj, key or elemId) -> tuple of (opId, kind); kind: 'v', 'c' (counter) or a type
        self.elems = {}                       # list / text obj -> every elemId ever inserted
        self.keys = {'_root': []}             # map / table obj -> every key ever written

    def get_live(self, obj, key):
        return self.live.get((obj, key), ())

    def apply(self, op, op_id):
        """one op (already expanded: no multi-insert) with its opId"""
        obj, act = op['obj'], op['action']
        if act == 'inc':
            return
        if op.get('insert'):
            key = op_id
            self.elems[obj].append(op_id)
        elif 'key' in op:
            key = op['key']
            if key not in self.live_keys(obj):
                self.keys[obj].append(key)
        else:
            key = op['elemId']
        preds = set(op.get('pred', ()))
        live = tuple(x for x in self.get_live(obj, key) if x[0] not in preds)
        if act == 'del':
            pass
        elif act in TYPES:
            live += ((op_id, TYPES[act]),)
            self.types[op_id] = TYPES[act]
            self.objs.append(op_id)
            if TYPES[act] in ('list', 'text'):
                self.elems[op_id] = []
            else:
                self.keys[op_id] = []
        else:
            live += ((op_id, 'c' if op.get('datatype') == 'counter' else 'v'),)
        self.live[(obj, key)] = live

    def live_keys(self, obj):
        return self.keys[obj]


class View(Model):
    """A writer's model: the round's snapshot plus its own ops so far (copy on write)."""

    def __init__(self, base):   # noqa: super().__init__ not called: every table is an overlay of base's
        self.base = base
        self.types, self.live, self.elems, self.keys = dict(), dict(), dict(), dict()
        self.objs = []    # objects this writer made

    def get_live(self, obj, key):
        k = (obj, key)
        return self.live[k] if k in self.live else self.base.live.get(k, ())

    def type_of(self, obj):
        return self.types.get(obj) or self.base.types[obj]

    def apply(self, op, op_id):
        obj = op['obj']
        if op.get('insert') and obj not in self.elems:
            self.elems[obj] = list(self.base.elems[obj])
        if 'key' in op and obj not in self.keys:
            self.keys[obj] = list(self.base.keys[obj])
        Model.apply(self, op, op_id)

    def elems_of(self, obj):
        return self.elems[obj] if obj in self.elems else self.base.elems[obj]

    def keys_of(self, obj):
        return self.keys[obj] if obj in self.keys else self.base.keys[obj]

    def live_keys(self, obj):
        return self.keys_of(obj)

    def all_objs(self):
        return self.base.objs + self.objs


class _Writer:
    """the ops of one change by `actor`, starting at counter `start`"""

    def __init__(self, gen, view, actor, start):
        self.g, self.rnd, self.v, self.actor, self.op, self.ops = gen, gen.rnd, view, actor, start, []

    def emit(self, op):
        op_id = '%d@%s' % (self.op, self.actor)
        self.op += 1
        self.ops.append(op)
        self.v.apply(op, op_id)
        return op_id

    # ---- values
    def scalar(self):
        r = self.rnd.random()
        if r < 0.4:
            return {'value': self.rnd.choice(('x', 'yy', 'ünï', '🐦', '')) + str(self.rnd.randrange(100))}
        if r < 0.6:
            return {'value': self.rnd.randrange(-1000, 1000)}
        if r < 0.7:
            return {'value': self.rnd.choice((True, False, None))}
        if r < 0.8:
            return {'value': self.rnd.randrange(0, 500), 'datatype': self.rnd.choice(('uint', 'timestamp'))}
        if r < 0.85:
            return {'value': self.rnd.randrange(-9, 9) / 4, 'datatype': 'float64'}
        return {'value': self.rnd.randrange(-20, 20), 'datatype': 'counter'}

    # ---- picking targets
    def pick_obj(self, kinds):
        objs = self.v.all_objs()
        cands = [o for o in objs[-400:] if self.v.type_of(o) in kinds]
        if self.rnd.random() < 0.3:
            cands = [o for o in objs if self.v.type_of(o) in kinds]
        return self.rnd.choice(cands) if cands else None

    def pick_key(self, obj):
        keys = self.v.keys_of(obj)
        r = self.rnd.random()
        if r < 0.5 or not keys:
            return self.rnd.choice(HOT_KEYS) if r < 0.35 or not keys else 'k%d' % self.rnd.randrange(40)
        return self.rnd.choice(keys)

    def make_action(self):
        if not self.g.room():
            return None
        return self.rnd.choice(('makeMap', 'makeList', 'makeText', 'makeTable', 'makeMap', 'makeList'))

    # ---- map / table keys
    def map_write(self, obj=None, key=None):
        obj = obj or self.pick_obj(('map', 'table'))
        key = key or self.pick_key(obj)
        live = self.v.get_live(obj, key)
        pred = [x[0] for x in live]
        r = self.rnd.random()
        counters = [x[0] for x in live if x[1] == 'c']
        if counters and r < 0.3:
            self.emit({'action': 'inc', 'obj': obj, 'key': key, 'value': self.rnd.randrange(-5, 9), 'pred': [self.rnd.choice(counters)]})
        elif live and r < 0.4:
            self.emit({'action': 'del', 'obj': obj, 'key': key, 'pred': pred})
        elif r < 0.55 and self.make_action():
            # set, then make* over it in the same change
            s = self.emit(dict({'action': 'set', 'obj': obj, 'key': key, 'pred': pred}, **self.scalar()))
            child = self.emit({'action': self.make_action() or 'makeMap', 'obj': obj, 'key': key, 'pred': [s]})
            self.fill(child)
        elif r < 0.75 and self.make_action():
            child = self.emit({'action': self.make_action(), 'obj': obj, 'key': key, 'pred': pred})
            if self.rnd.random() < 0.7:
                self.fill(child)
        else:
            self.emit(dict({'action': 'set', 'obj': obj, 'key': key, 'pred': pred}, **self.scalar()))

    # ---- lists and texts
    def insert_run(self, obj, n, ref=None):
        elems = self.v.elems_of(obj)
        if ref is None:
            ref = self.rnd.choice(elems) if elems and self.rnd.random() < 0.85 else '_head'
        text = self.v.type_of(obj) == 'text'
        for _ in range(n):
            if text:
                op = {'value': self.rnd.choice('abcdefgh ünï🐦')}
            elif self.rnd.random() < 0.12 and self.make_action():
                child = self.emit({'action': self.make_action(), 'obj': obj, 'elemId': ref, 'insert': True, 'pred': []})
                if self.rnd.random() < 0.5:
                    self.fill(child)
                ref = child
                continue
            else:
                op = self.scalar()
            ref = self.emit(dict({'action': 'set', 'obj': obj, 'elemId': ref, 'insert': True, 'pred': []}, **op))
        return ref

    def list_edit(self, obj):
        elems = [e for e in self.v.elems_of(obj)[-300:] if self.v.get_live(obj, e)]
        if not elems:
            self.insert_run(obj, self.rnd.randint(1, 8))
            return
        e = self.rnd.choice(elems)
        live = self.v.get_live(obj, e)
        pred = [x[0] for x in live]
        r = self.rnd.random()
        counters = [x[0] for x in live if x[1] == 'c']
        if counters and r < 0.3:
            self.emit({'action': 'inc', 'obj': obj, 'elemId': e, 'value': self.rnd.randrange(1, 9), 'pred': [self.rnd.choice(counters)]})
        elif r < 0.55:
            self.emit({'action': 'del', 'obj': obj, 'elemId': e, 'pred': pred})
        elif r < 0.7 and self.v.type_of(obj) == 'list' and self.make_action():
            child = self.emit({'action': self.make_action(), 'obj': obj, 'elemId': e, 'pred': pred})
            self.fill(child)
        else:
            op = {'value': self.rnd.choice('XYZ')} if self.v.type_of(obj) == 'text' else self.scalar()
            self.emit(dict({'action': 'set', 'obj': obj, 'elemId': e, 'pred': pred}, **op))

    def two_texts(self):
        """insert runs alternating between two lists / texts in one change: typing runs that must not join across objects"""
        cands = [o for o in self.v.all_objs()[-200:] if self.v.type_of(o) in ('text', 'list')]
        if len(cands) < 2:
            return
        a, b = self.rnd.sample(cands, 2)
        ra = rb = None
        for _ in range(self.rnd.randint(2, 6)):
            ra = self.insert_run(a, self.rnd.randint(1, 4), ra)
            rb = self.insert_run(b, self.rnd.randint(1, 4), rb)

    # ---- objects
    def fill(self, obj):
        """a few ops into an object made earlier in this change"""
        t = self.v.type_of(obj)
        for _ in range(self.rnd.randint(0, 3)):
            if t in ('list', 'text'):
                self.insert_run(obj, self.rnd.randint(1, 8))
            elif t == 'table':
                self.table_row(obj)
            else:
                self.map_write(obj, 'k%d' % self.rnd.randrange(6))

    def table_row(self, table):
        row = self.emit({'action': 'makeMap', 'obj': table, 'key': '%08x-row' % self.rnd.getrandbits(32), 'pred': []})
        for f in self.rnd.sample(('title', 'done', 'n', 'tag'), self.rnd.randint(1, 3)):
            self.emit(dict({'action': 'set', 'obj': row, 'key': f, 'pred': []}, **self.scalar()))

    def chain(self, depth, start=None):
        """nesting `depth` levels deep, alternating list and map; an edit at the bottom"""
        obj = start or self.pick_obj(('map', 'list'))
        for _ in range(depth):
            if self.v.type_of(obj) == 'list':
                elems = self.v.elems_of(obj)
                ref = elems[-1] if elems and self.rnd.random() < 0.7 else '_head'
                obj = self.emit({'action': 'makeMap', 'obj': obj, 'elemId': ref, 'insert': True, 'pred': []})
            else:
                key = 'n%d' % self.rnd.randrange(3)
                obj = self.emit({'action': 'makeList', 'obj': obj, 'key': key, 'pred': [x[0] for x in self.v.get_live(obj, key)]})
        if self.v.type_of(obj) == 'list':
            self.insert_run(obj, 2)
        else:
            self.map_write(obj, 'leaf')
        return obj

    def random_action(self):
        r = self.rnd.random()
        if r < 0.25:
            self.map_write()
        elif r < 0.5:
            obj = self.pick_obj(('list', 'text'))
            if obj is None:
                self.map_write(key=None)
            else:
                self.insert_run(obj, self.rnd.randint(1, 8))
        elif r < 0.68:
            obj = self.pick_obj(('list', 'text'))
            if obj is not None:
                self.list_edit(obj)
        elif r < 0.76:
            self.two_texts()
        elif r < 0.84:
            # a new object, then ops into it in the same change
            obj, act = self.pick_obj(('map',)), self.make_action()
            if act:
                key = self.pick_key(obj)
                self.fill(self.emit({'action': act, 'obj': obj, 'key': key, 'pred': [x[0] for x in self.v.get_live(obj, key)]}))
        elif r < 0.9:
            table = self.pick_obj(('table',))
            if table is not None:
                self.table_row(table)
        elif r < 0.94 and self.g.room():
            self.chain(self.rnd.randint(2, max(2, min(self.g.depth, 12))))
        else:
            obj = self.pick_obj(('map', 'table', 'list', 'text'))
            if obj is not None and self.v.type_of(obj) in ('list', 'text'):
                self.list_edit(obj)
            elif obj is not None:
                self.map_write(obj)


class ObjGen:
    """
    actors      number of replicas (1-8)
    rounds      rounds of concurrent writing
    objects     the generator stops making objects once about this many exist (forced shapes excepted)
    actions     actions per change: 1..actions
    big_lists   chance per change of one long insert burst (50-600 elements) into a list or text
    depth       deepest list / map nesting one forced round builds
    boundary    open with lists of exactly 2 047 .. 4 097 rows and tiny objects between them
    """

    def __init__(self, seed, actors=3, rounds=40, objects=200, actions=4, big_lists=0.02, depth=50, boundary=False):
        self.rnd = random.Random(seed)
        self.actor_ids = sorted('%032x' % self.rnd.getrandbits(128) for _ in range(actors))
        self.rounds, self.objects, self.actions, self.big_lists, self.depth, self.boundary = rounds, objects, actions, big_lists, depth, boundary
        self.model = Model()
        self.changes, self.hashes = [], []
        self.round_starts = []                # index into changes of each round's first change
        self.heads, self.max_op, self.seq = [], 0, {a: 0 for a in self.actor_ids}
        self.contested = []

    def room(self):
        return len(self.model.objs) < self.objects

    def _round(self, plans):
        """plans: [(actor, fn(writer))]; every writer sees the model as it is now"""
        start, deps, written = self.max_op + 1, sorted(self.heads), []
        self.round_starts.append(len(self.changes))
        for actor, plan in plans:
            w = _Writer(self, View(self.model), actor, start)
            plan(w)
            if not w.ops:
                continue
            self.seq[actor] += 1
            ch = {'actor': actor, 'seq': self.seq[actor], 'startOp': start, 'time': self.rnd.randrange(0, 2 ** 33) if self.rnd.random() < 0.3 else 0,
                  'message': self.rnd.choice(('', '', 'edit')), 'deps': deps, 'ops': w.ops}
            data, h = columnar.encode_change_raw(ch)   # DEFLATEd from 256 bytes, as the reference's encoder does
            self.changes.append(data)
            self.hashes.append(h)
            written.append((w.ops, start, actor, h))
        for ops, first, actor, _ in written:
            for i, op in enumerate(ops):
                self.model.apply(op, '%d@%s' % (first + i, actor))
            self.max_op = max(self.max_op, first + len(ops) - 1)
        if written:
            self.heads = [h for *_, h in written]

    def _random_plan(self, w):
        for _ in range(self.rnd.randint(1, self.actions)):
            w.random_action()
        if self.rnd.random() < self.big_lists:
            obj = w.pick_obj(('list', 'text'))
            if obj is not None:
                for _ in range(self.rnd.randint(10, 100)):
                    w.insert_run(obj, self.rnd.randint(1, 8))

    def _boundary_plan(self, w):
        for rows in BOUNDARY_ROWS:
            lst = w.emit({'action': self.rnd.choice(('makeList', 'makeText')), 'obj': '_root', 'key': 'big%d' % rows, 'pred': []})
            left = rows
            while left:
                n = min(left, self.rnd.randint(1, 8))
                w.insert_run(lst, n) if w.v.type_of(lst) == 'text' else self._plain_run(w, lst, n)
                left -= n
            for i in range(self.rnd.randint(1, 4)):   # tiny objects between the big ones
                t = w.emit({'action': self.rnd.choice(('makeList', 'makeMap', 'makeText')), 'obj': '_root', 'key': 'tiny%d-%d' % (rows, i), 'pred': []})
                if w.v.type_of(t) == 'map':
                    w.emit({'action': 'set', 'obj': t, 'key': 'v', 'value': i, 'pred': []})
                else:
                    self._plain_run(w, t, self.rnd.randint(1, 2))

    def _plain_run(self, w, obj, n):
        """n scalar inserts after one random element (no objects: the row count is exact)"""
        elems = w.v.elems_of(obj)
        ref = self.rnd.choice(elems) if elems else '_head'
        for _ in range(n):
            v = 'c' if w.v.type_of(obj) == 'text' else self.rnd.randrange(100)
            ref = w.emit({'action': 'set', 'obj': obj, 'elemId': ref, 'insert': True, 'value': v, 'pred': []})

    def _contest(self, key):
        """every actor makes an object on `key` at the same counter"""
        def plan(w):
            w.emit({'action': self.rnd.choice(('makeMap', 'makeList', 'makeText', 'makeTable')), 'obj': '_root', 'key': key,
                    'pred': [x[0] for x in w.v.get_live('_root', key)]})
        self._round([(a, plan) for a in self.actor_ids])
        self.contested = [x[0] for x in self.model.get_live('_root', key) if x[1] not in ('v', 'c')]

    def _edit_inside(self, w, objs):
        for o in objs:
            t = w.v.type_of(o)
            if t in ('list', 'text'):
                w.insert_run(o, self.rnd.randint(1, 3))
            elif t == 'table':
                w.table_row(o)
            else:
                w.map_write(o, 'k%d' % self.rnd.randrange(3))

    def _writers(self):
        k = self.rnd.randint(1, len(self.actor_ids))
        return sorted(self.rnd.sample(self.actor_ids, k))

    def generate(self):
        if self.boundary:
            self._round([(self.actor_ids[0], self._boundary_plan)])
        forced = {max(1, self.rounds // 5): 'contest', max(2, self.rounds // 2): 'deep', max(3, (3 * self.rounds) // 4): 'scalar_vs_object'}
        r = 0
        while r < self.rounds:
            what = forced.get(r)
            if what == 'contest':
                self._contest('contested')
                # edits inside each object, while one actor overwrites the key with a scalar ...
                over = self.actor_ids[-1]
                self._round([(a, lambda w: self._edit_inside(w, self.contested)) for a in self.actor_ids[:-1]] +
                            [(over, lambda w: w.emit({'action': 'set', 'obj': '_root', 'key': 'contested', 'value': 'plain',
                                                      'pred': [x[0] for x in w.v.get_live('_root', 'contested')]}))])
                # ... after the overwrite, and after a delete
                self._round([(a, lambda w: self._edit_inside(w, self.contested)) for a in self.actor_ids])
                self._round([(self.actor_ids[0], lambda w: w.emit({'action': 'del', 'obj': '_root', 'key': 'contested',
                                                                   'pred': [x[0] for x in w.v.get_live('_root', 'contested')]}))])
                self._round([(a, lambda w: self._edit_inside(w, self.contested)) for a in self.actor_ids])
                r += 5
            elif what == 'deep':
                bottom = {}
                self._round([(self.actor_ids[0], lambda w: bottom.setdefault('o', w.chain(self.depth, '_root')))])
                self._round([(a, lambda w: self._edit_inside(w, [bottom['o']])) for a in self._writers()])
                r += 2
            elif what == 'scalar_vs_object':
                # one actor: set then make* on key 'b'; the others set 'b' concurrently; later, edits inside the object
                def mk(w):
                    s = w.emit(dict({'action': 'set', 'obj': '_root', 'key': 'b', 'pred': [x[0] for x in w.v.get_live('_root', 'b')]}, **w.scalar()))
                    w.emit({'action': self.rnd.choice(('makeList', 'makeMap', 'makeText')), 'obj': '_root', 'key': 'b', 'pred': [s]})
                plans = [(self.actor_ids[0], mk)] + [(a, lambda w: w.map_write('_root', 'b')) for a in self.actor_ids[1:]]
                self._round(plans)
                objs = [x[0] for x in self.model.get_live('_root', 'b') if x[1] not in ('v', 'c')]
                self._round([(a, lambda w: self._edit_inside(w, objs)) for a in self._writers()])
                r += 2
            else:
                self._round([(a, self._random_plan) for a in self._writers()])
                r += 1
        return self.changes


def generate(seed, **knobs):
    return ObjGen(seed, **knobs).generate()
