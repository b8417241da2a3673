// amgpu — kernels #4: patch emission.
//
// Replaces (reference paths relative to /root/reference):
//   backend/new.js:884-1040   updatePatchProperty   backend/new.js:747-782  appendEdit (run coalescing)
//   backend/new.js:1461-1528  setupPatches          backend/new.js:1604-1635 documentPatch (getPatch)
//
// The reference's incremental patch is an edit log in application order whose list indexes are valid
// at the moment each edit is appended. For an op applied at time t on the element at document
// position p the index is  #{elements e of the same list : pos_e < p, t_ins(e) < t, t_del(e) > t}.
// That is an offline dominance count; it is computed for all ops at once by a most-significant-bit
// first radix partition over the time bits (DominanceLevelKernel): items (element insertions +1,
// first deletions -1, and one query per op) start in (object, position) order; at bit b every query
// with bit b set adds the weighted count of bit-b-clear points that precede it inside its current
// group (same higher time bits, same list), then the group is stably split on bit b.
// Supported in incremental mode: map/table objects (set/del/make*, conflicts) and list/text objects
// whose touched elements carry only their insert row (insert + delete; no element updates, no nested
// objects inside lists, no counters). Anything else raises AMG_ERR_UNSUPPORTED — there is no CPU path.
#pragma once
#include "opset.cuh"

namespace amg {

// flat patch records (copied to the host verbatim)
struct PropRec { u64 obj, opId; u32 keyOff, keyLen, valLen, valOff, flags /* action<<8 | 1 = empty key | 2 = counter: value is the int64 (pad:valOff) */, pad; };
struct EditRec { u64 obj, opId; u32 index, kind /* 0 insert 1 remove 2 update | runStart<<8 | action<<16 */, valLen, valOff; };
enum { EK_INSERT = 0, EK_REMOVE = 1, EK_UPDATE = 2 };
enum { EF_POP = 0x400, EF_GROUP_FIRST = 0x800, EF_START = 0x100, EF_MULTI = 0x200, EF_COUNTER = 0x1000 /* value = int64 (valOff:valLen), not arena bytes */ };

// The bytes the patch records point at (map keys, value payloads) travel inside the patch: counted per record, laid out by
// a prefix sum, copied from the arena; the records' offsets are rewritten to positions in the patch buffer. (The host no
// longer needs a mirror of the arena to read a patch.)
struct PatchBytesCountKernel {
  const PropRec* props; size_t numProps; const EditRec* edits; u32* len;
  HD void operator()(size_t i) const {
    if (i < numProps) { const PropRec& r = props[i]; len[i] = (r.keyLen == 0xffffffffu ? 0u : r.keyLen) + ((r.flags & 2u) ? 0u : (r.valLen >> 4)); }
    else { const EditRec& r = edits[i - numProps]; len[i] = (r.kind & EF_COUNTER) ? 0u : (r.valLen >> 4); }
  }
};
struct PatchBytesGatherKernel {
  const u8* arena; PropRec* props; size_t numProps; EditRec* edits; const u32* off; u32 bytesOff /* of the section inside the patch */; u8* out; u64* errWord;
  // decodeValue (columnar.js:300-329) runs in the reference whenever a value reaches a patch: numbers must be complete
  // LEB128 values within 53 bits, floating point payloads must be 8 bytes
  HD void validate(u32 valLen, u32 valOff, size_t i) const {
    if (const u32 e = decode_value_error(arena, valLen, valOff)) raise(errWord, e, i);
  }
  HD void operator()(size_t i) const {
    u32 at = off[i];
    if (i < numProps) {
      PropRec& r = props[i];
      if (r.keyLen != 0xffffffffu) { for (u32 k = 0; k < r.keyLen; k++) out[at + k] = arena[r.keyOff + k]; r.keyOff = bytesOff + at; at += r.keyLen; }
      if (!(r.flags & 2u)) { const u32 n = r.valLen >> 4; if (!(r.flags & 1u) && (r.flags >> 8) == 1) validate(r.valLen, r.valOff, i); for (u32 k = 0; k < n; k++) out[at + k] = arena[r.valOff + k]; r.valOff = bytesOff + at; }
    } else {
      EditRec& r = edits[i - numProps];
      if (!(r.kind & EF_COUNTER)) { const u32 n = r.valLen >> 4; if ((r.kind & 0xff) != EK_REMOVE && (r.kind >> 16) == 1) validate(r.valLen, r.valOff, i); for (u32 k = 0; k < n; k++) out[at + k] = arena[r.valOff + k]; r.valOff = bytesOff + at; }
    }
  }
};

// ---------------------------------------------------------------- per-position state in document order
struct GroupHeadKernel {   // group = rows of one map key / one list element (insert row + its update rows), adjacent in document order
  const u8* arena; DocRows d; u32* head;
  HD void operator()(size_t p) const {
    bool h = p == 0 || d.obj[p] != d.obj[p - 1];
    if (!h) {
      const bool listA = d.keyStrLen[p] == NULL32, listB = d.keyStrLen[p - 1] == NULL32;
      if (listA != listB) h = true;
      else if (listA) h = (d.flags[p] & F_INSERT) != 0;
      else {
        h = d.keyStrLen[p] != d.keyStrLen[p - 1];
        for (u32 i = 0; !h && i < d.keyStrLen[p]; i++) h = arena[d.keyStrOff[p] + i] != arena[d.keyStrOff[p - 1] + i];
      }
    }
    head[p] = h ? 1u : 0u;
  }
};
struct GroupStatsKernel {   // group id = inclusive scan of heads - 1; counts rows and visible rows per group
  const u32* headScan /* exclusive scan of head */; const u32* head; const u32* succCnt; DocRows d; u32* groupOf; u32* groupRows; u32* groupVisible; u32* groupFirst; u64* errWord; int allowCounters;
  u32* groupHasChild /* some visible row of the group is a make* op */;
  HD void operator()(size_t p) const {
    const u32 g = headScan[p] + head[p] - 1; groupOf[p] = g;
    atomic_add(&groupRows[g], 1u);
    if (succCnt[p] == 0) { atomic_add(&groupVisible[g], 1u); const u32 a = flags_action(d.flags[p]); if (a % 2 == 0 && a != ACT_DEL) groupHasChild[g] = 1; }
    if (head[p]) groupFirst[g] = (u32)p;

  }
};

// ---------------------------------------------------------------- incremental: touched groups / objects
struct TouchKernel {   // new rows and the targets of new succ entries touch their group and object (objTouchedAt = earliest such time)
  DocRows d; const u32* groupOf; const u32* firstNewSucc; u32* groupTouched; u32* objTouchedAt /* per position of the object's make row; 0xffffffff = untouched */;
  const u32* objPos /* per position: position of the object's make row or ROW_NONE (root) */; u32* rootTouched;
  HD void operator()(size_t p) const {
    if (d.time[p] == 0 && firstNewSucc[p] == 0xffffffffu) return;
    groupTouched[groupOf[p]] = 1;
    u32 t = firstNewSucc[p]; if (d.time[p] != 0 && d.time[p] < t) t = d.time[p];
    if (objPos[p] == ROW_NONE) *rootTouched = 1; else warp_agg_min_at(objTouchedAt, objPos[p], t);   // all rows of one object meet here: one atomic per warp
  }
};
// setupPatches (new.js:1461-1528): a touched object links itself into its parent (the group of its make row), recursively.
// Objects are visited in the order they were first touched; the time travels up with the link so that link edits on a
// list parent can be ordered the same way. A list element that already carries edits of this call needs no link edit.
// When the key / element was itself touched by this call, the parent's patch already holds the child (patchExists,
// new.js:1472-1474, 1509-1510) and the climb stops there: the parent's ancestors are linked at the parent's own time
// (or a later child's), not at this child's.
struct LinkKernel {
  DocRows d; const u32* groupOf; const u32* groupHasChild; const u32* groupFirst; const u32* groupTouched; const u32* objPos; u32* groupLinked; u32* objTouchedAt; u32* rootTouched; u32* linkDone; u32* changed;
  u32* listLinkTime /* per position of an element's insert row; 0xffffffff = none */; u32* anyListLink;
  HD void operator()(size_t p) const {
    const u32 t = objTouchedAt[p];
    if (t == 0xffffffffu || linkDone[p] == t) return;
    linkDone[p] = t; *changed = 1;
    const u32 g = groupOf[p];
    // hasChildren (new.js:1465,1521): objectMeta.children of a key / element is only kept up to date while one of its
    // visible values is an object (new.js:919-935), so an object that was overwritten by plain values links nothing.
    // (Not modelled: the reference also keeps a snapshot alive while the lowest-id value stays visible after the last
    // object value went away; that depends on the order of earlier calls.)
    if (groupHasChild[g] == 0) return;
    if (d.keyStrLen[p] == NULL32) {     // child object inside a list: an update edit per visible value unless the element has edits already
      const u32 e = groupFirst[g];
      atomic_min(&listLinkTime[e], t); *anyListLink = 1;   // whether an edit is really needed is known once the pops are replayed (elemHasLive)
    } else groupLinked[g] = 1;
    if (groupTouched[g]) return;
    if (objPos[p] == ROW_NONE) *rootTouched = 1; else atomic_min(&objTouchedAt[objPos[p]], t);
  }
};
// ---------------------------------------------------------------- which conflicting values the reference re-emits
// mergeDocChangeOps (new.js:1085-1138) processes the change ops of one author in "groups" (consecutive ops on the
// same key that do not overwrite each other). After a group's last op is placed, the remaining document ops of
// that key (those with a greater opId) are only re-emitted into the patch if no further group could be gathered
// into the same pass (new.js:1119-1129, 1149); otherwise they are passed over silently (new.js:1225-1230). The
// patch content of a key is what the LAST pass touching it emitted (props[key] is reset per pass, new.js:1037).
HD int key_cmp_utf16(const u8* a, u32 la, const u8* b, u32 lb) {   // JS string `<` on UTF-8 bytes
  const u32 n = la < lb ? la : lb;
  for (u32 i = 0; i < n; i++) {
    u32 x = a[i], y = b[i];
    if (x != y) {
      if (x == 0xEE || x == 0xEF) x += 5; else if (x >= 0xF0 && x <= 0xF4) x -= 2;
      if (y == 0xEE || y == 0xEF) y += 5; else if (y >= 0xF0 && y <= 0xF4) y -= 2;
      return x < y ? -1 : 1;
    }
  }
  return la < lb ? -1 : (la > lb ? 1 : 0);
}
struct OpAtTimeKernel { const u32* time; u32* opAt; HD void operator()(size_t i) const { opAt[time[i] - 1] = (u32)i; } };
struct MapGroupCtx {
  const u8* arena; OpRows ops; const u32* opAt; size_t numOps; const u32* passOf /* per batch change: pass of the causal gate */;
  HD bool samePass(u32 i, u32 j) const { return passOf[ops.change[i]] == passOf[ops.change[j]]; }   // every pass is its own applyOps run (new.js:1822-1841)
  HD bool isMapOp(u32 i) const { return ops.keyStrLen[i] != NULL32; }
  HD bool sameKey(u32 i, u32 j) const {
    if (ops.keyStrLen[i] != ops.keyStrLen[j]) return false;
    for (u32 k = 0; k < ops.keyStrLen[i]; k++) if (arena[ops.keyStrOff[i] + k] != arena[ops.keyStrOff[j] + k]) return false;
    return true;
  }
  HD bool sameRun(u32 i, u32 j) const {   // ops that one mergeDocChangeOps call may gather onto one key / list element
    if (id_actor(ops.id[i]) != id_actor(ops.id[j]) || ((ops.flags[i] ^ ops.flags[j]) & F_INSERT) != 0 || ops.obj[i] != ops.obj[j] || isMapOp(i) != isMapOp(j) || !samePass(i, j)) return false;
    if (isMapOp(i)) return sameKey(i, j);
    return (ops.flags[i] & F_INSERT) == 0 && ops.key[i] == ops.key[j];
  }
};
struct RunHeadKernel { MapGroupCtx c; u32* runHead; HD void operator()(size_t t) const { runHead[t] = (t == 0 || !c.sameRun(c.opAt[t], c.opAt[t - 1])) ? 1u : 0u; } };
struct GroupSplitKernel {   // one thread per run: a new group starts where an op overwrites an op of the current group (new.js:1092-1101)
  MapGroupCtx c; const u32* runHead; u32* groupHead;
  HD void operator()(size_t t0) const {
    if (!runHead[t0]) return;
    size_t gstart = t0; groupHead[t0] = 1;
    for (size_t t = t0 + 1; t < c.numOps && !runHead[t]; t++) {
      const u32 i = c.opAt[t]; bool over = false;
      for (u32 j = 0; j < c.ops.predNum[i] && !over; j++) {
        const u64 p = c.ops.predId[c.ops.predOff[i] + j];
        for (size_t u = gstart; u < t && !over; u++) over = c.ops.id[c.opAt[u]] == p;
      }
      groupHead[t] = over ? 1u : 0u;
      if (over) gstart = t;
    }
  }
};
struct GroupFinalKernel {   // pass 0: finalTime[g] = latest group on key group g; pass 1: that group publishes bound / failed / members
  int pass; MapGroupCtx c; const u32* groupHead; IdTable t; const u32* rowOfOp; const u32* pos; const u32* groupOf; DocRows w; Ord ord;
  u32* finalTime; u64* bound; u32* failed; u32* member;
  HD void operator()(size_t t0) const {
    if (!groupHead[t0]) return;
    const u32 i0 = c.opAt[t0]; if (!c.isMapOp(i0)) return;
    u64 b = 0; u32 g = ROW_NONE; size_t t = t0;
    for (; t < c.numOps && (t == t0 || !groupHead[t]); t++) {
      const u32 i = c.opAt[t];
      if (flags_action(c.ops.flags[i]) == ACT_DEL) {
        for (u32 j = 0; j < c.ops.predNum[i]; j++) {
          const u32 target = id_lookup(this->t, c.ops.predId[c.ops.predOff[i] + j]); if (target == ROW_NONE) continue;
          const u64 o = ord(w.id[target]); if (o > b) b = o; g = groupOf[pos[target]];
        }
      } else {
        const u64 o = ord(c.ops.id[i]); if (o > b) b = o;
        if (rowOfOp[i] != ROW_NONE) { g = groupOf[pos[rowOfOp[i]]]; if (pass == 1 && finalTime[g] == (u32)t0 + 1) member[pos[rowOfOp[i]]] = 1; }
      }
    }
    if (g == ROW_NONE) return;
    if (pass == 0) { atomic_max(&finalTime[g], (u32)t0 + 1); return; }
    if (finalTime[g] != (u32)t0 + 1) return;
    bool gathered = false;
    if (t < c.numOps) {
      const u32 nx = c.opAt[t];
      gathered = c.isMapOp(nx) && c.samePass(nx, i0) && id_actor(c.ops.id[nx]) == id_actor(c.ops.id[i0]) && ((c.ops.flags[nx] ^ c.ops.flags[i0]) & F_INSERT) == 0 && c.ops.obj[nx] == c.ops.obj[i0] &&
                 key_cmp_utf16(c.arena + c.ops.keyStrOff[i0], c.ops.keyStrLen[i0], c.arena + c.ops.keyStrOff[nx], c.ops.keyStrLen[nx]) < 0;
    }
    bound[g] = b; failed[g] = gathered ? 0u : 1u;
    // members of a group that straddles the walk above were flagged on the fly; flag again now that finalTime is known
    for (size_t u = t0; u < t; u++) { const u32 i = c.opAt[u]; if (rowOfOp[i] != ROW_NONE) member[pos[rowOfOp[i]]] = 1; }
  }
};
// What `counterState.value += decodeValue(...).value` (new.js:944, 954) adds for a value of the given tag: the number; JavaScript
// turns null / false into 0 and true into 1 (only invalid input carries those; anything else - float, string, bytes - is refused
// by IncCheckKernel before it gets here).
HD long long counter_operand(const u8* arena, u32 valLen, u32 valOff) {
  const u32 tag = valLen & 15;
  if (tag == 2) return 1;
  if (tag < 2) return 0;
  ByteReader br(arena, valOff, valOff + (valLen >> 4));
  return tag == 3 ? (long long)br.uleb() : br.sleb();
}
// A counter's total is a JavaScript number in the reference: the operands (53-bit integers, exact in a double) are added
// as doubles, in document order - the counter's `set` row first, then its increments by opId - so a total past 2^53 is
// rounded at each step exactly as the reference rounds it. The patch carries the total as an int64, which holds every
// such double in [-2^63, 2^63); a total outside that range is refused (KE_COUNTER_RANGE, DESIGN.md section 5).
HD u64 counter_bits(double v) { u64 b; memcpy(&b, &v, 8); return b; }
HD bool counter_int64(u64 bits, long long* out) {
  double v; memcpy(&v, &bits, 8);
  if (!(v >= -9223372036854775808.0 && v < 9223372036854775808.0)) return false;
  *out = (long long)v; return true;
}
// Counters (new.js:941-966): increments are successors of the `set` that created the counter. The counter shows with the
// summed value once every successor turned out to be an `inc`; the reference emits it while processing the last of them.
struct CounterKernel {
  const u8* arena; DocRows d; const u32* succOff; const u64* succ; const u32* groupOf; const u32* groupFirst; const u32* groupRows;
  u32* counterLast /* position of the last inc row, ROW_NONE = not a visible counter */; u64* counterTotal /* double bits */; u32* counterOwner /* per inc row that completes a counter: the counter's row */;
  HD long long valueOf(u32 r) const { return counter_operand(arena, d.valLen[r], d.valOff[r]); }
  HD void operator()(size_t p) const {
    counterLast[p] = ROW_NONE;
    if (flags_action(d.flags[p]) != ACT_SET || (d.valLen[p] & 15) != 8) return;
    const u32 s0 = succOff[p], s1 = succOff[p + 1]; if (s0 == s1) return;
    const u32 g = groupOf[p], gf = groupFirst[g], rows = groupRows[g];
    u32 last = 0;
    for (u32 s = s0; s < s1; s++) {
      u32 r = ROW_NONE;
      for (u32 q = gf; q < gf + rows; q++) if (d.id[q] == succ[s]) { r = q; break; }
      if (r == ROW_NONE || flags_action(d.flags[r]) != ACT_INC) return;   // deleted or overwritten: the counter is gone
      if (r > last) last = r;
    }
    double total = (double)valueOf((u32)p);
    for (u32 q = (u32)p + 1; q <= last; q++) {   // the increments in row (= opId) order
      bool mine = false; for (u32 s = s0; s < s1 && !mine; s++) mine = d.id[q] == succ[s];
      if (mine) total += (double)valueOf(q);
    }
    counterLast[p] = last; counterTotal[p] = counter_bits(total); counterOwner[last] = (u32)p;
  }
};
struct PropFlagKernel {   // which positions emit a prop record
  DocRows d; const u32* groupOf; const u32* groupTouched; const u32* groupLinked; const u32* succCnt; int wholeDoc;
  const u32* finalTime; const u64* bound; const u32* failed; const u32* member; Ord ord; u32* emit; u32* groupEmitted; const u32* counterLast;
  HD void operator()(size_t p) const {
    u32 e = 0;
    if (d.keyStrLen[p] != NULL32) {
      // q = the row whose processing puts this value into the patch: the row itself, or a counter's last increment
      u32 q = ROW_NONE;
      if (counterLast[p] != ROW_NONE) q = counterLast[p]; else if (succCnt[p] == 0 && flags_action(d.flags[p]) != ACT_INC) q = (u32)p;
      if (q != ROW_NONE) {
        const u32 g = groupOf[p];
        if (wholeDoc) e = 1;
        else if (groupTouched[g]) e = (finalTime[g] == 0 || failed[g] || member[q] || ord(d.id[q]) <= bound[g]) ? 1 : 0;
        else if (groupLinked[g]) e = 1;
      }
    }
    emit[p] = e;
    if (e) atomic_add(&groupEmitted[groupOf[p]], 1u);
  }
};
struct PropMarkerKernel {   // a touched key with nothing to show is reported as `key: {}` (new.js:1037)
  DocRows d; const u32* groupOf; const u32* groupTouched; const u32* head; const u32* groupEmitted; int wholeDoc; u32* emit; u32* marker;
  HD void operator()(size_t p) const {
    u32 m = 0;
    if (!wholeDoc && d.keyStrLen[p] != NULL32 && head[p] && groupTouched[groupOf[p]] && groupEmitted[groupOf[p]] == 0) { m = 1; emit[p] = 1; }
    marker[p] = m;
  }
};
struct PropEmitKernel {
  DocRows d; const u32* emit; const u32* marker; const u32* slot; PropRec* out; const u32* counterLast; const u64* counterTotal; u64* errWord;
  HD void operator()(size_t p) const {
    if (!emit[p]) return;
    PropRec r; r.obj = d.obj[p]; r.opId = d.id[p]; r.keyOff = d.keyStrOff[p]; r.keyLen = d.keyStrLen[p]; r.valLen = d.valLen[p]; r.valOff = d.valOff[p];
    r.flags = (flags_action(d.flags[p]) << 8) | (marker[p] ? 1u : 0u); r.pad = 0;
    if (!marker[p] && counterLast[p] != ROW_NONE) {   // summed counter value instead of arena bytes
      long long total = 0; if (!counter_int64(counterTotal[p], &total)) raise(errWord, KE_COUNTER_RANGE, p);
      r.flags |= 2u; r.valOff = (u32)(u64)total; r.pad = (u32)((u64)total >> 32);
    }
    out[slot[p]] = r;
  }
};

// ---------------------------------------------------------------- whole-document list edits (getPatch)
// Whole-document list edits (documentPatch, new.js:1604-1635, through updatePatchProperty with isWholeDoc): a row that
// carries a value (pv: visible set / make*, or the increment that completes a counter) inserts the element if it is
// the first event of the element, otherwise updates it. A visible row WITHOUT a value (an `inc` that does not complete
// its counter: deleted counter, or one of several increments) registers a `remove` when it comes first; a later value
// undoes it and is then reported as an update; with no later value the remove stays (reference behaviour, new.js:965 TODO).
struct ListRowClassKernel {
  DocRows d; const u32* groupOf; const u32* succCnt; const u32* counterOwner; u32* rowClass /* 0 nothing, 1 value, 2 visible without value */; u32* firstPv; u32* firstBare;
  HD void operator()(size_t p) const {
    u32 c = 0;
    if (d.keyStrLen[p] == NULL32) {
      const u32 a = flags_action(d.flags[p]);
      if (counterOwner[p] != ROW_NONE || (succCnt[p] == 0 && (a == ACT_SET || (a % 2 == 0 && a != ACT_DEL)))) c = 1;
      else if (succCnt[p] == 0) c = 2;
      if (c == 1) atomic_min(&firstPv[groupOf[p]], (u32)p); else if (c == 2) atomic_min(&firstBare[groupOf[p]], (u32)p);
    }
    rowClass[p] = c;
  }
};
struct ListVisFlagKernel {   // element visible (any visible row) flagged on the group head; emitting rows flagged individually
  DocRows d; const u32* groupOf; const u32* groupVisible; const u32* head; const u32* succCnt; u32* elemVis; u32* rowEmit;
  const u32* rowClass; const u32* firstPv; const u32* firstBare;   // null: link mode (plain visible rows only)
  HD void operator()(size_t p) const {
    const bool list = d.keyStrLen[p] == NULL32;
    elemVis[p] = (list && head[p] && groupVisible[groupOf[p]] > 0) ? 1u : 0u;   // an `inc` row counts as visible here, as in the reference (new.js:1622-1626)
    if (!rowClass) { rowEmit[p] = (list && succCnt[p] == 0) ? 1u : 0u; return; }
    const u32 g = groupOf[p];
    rowEmit[p] = (rowClass[p] == 1 || (rowClass[p] == 2 && firstBare[g] == (u32)p && firstPv[g] == 0xffffffffu)) ? 1u : 0u;
  }
};
struct ObjHeadKernel { DocRows d; u32* isObjHead; HD void operator()(size_t p) const { isObjHead[p] = (p == 0 || d.obj[p] != d.obj[p - 1]) ? 1u : 0u; } };
struct ObjStartKernel {   // objIdx = exclusive scan of heads (+head-1 fix-up); objStart[k] = first position of the k-th object
  const u32* isObjHead; u32* objIdx /* in: exclusive scan of isObjHead, out: object index */; u32* objStart; size_t n;
  HD void operator()(size_t p) const {
    const u32 k = objIdx[p] + isObjHead[p] - 1; objIdx[p] = k;
    if (isObjHead[p]) objStart[k] = (u32)p;
  }
};
struct DocEditEmitKernel {   // getPatch: visible rows of list objects in document order
  DocRows d; const u32* rowEmit; const u32* slot; const u32* elemVisScan /* exclusive */; const u32* objIdx; const u32* objStart;
  const u32* groupOf; const u32* groupFirst; const u32* rowClass; const u32* firstPv; const u32* firstBare; EditRec* out;
  const u32* counterOwner; const u64* counterTotal; u64* errWord;
  HD void operator()(size_t p) const {
    if (!rowEmit[p]) return;
    const u32 g = groupOf[p]; const u32 gp = groupFirst[g];
    const u32 src = counterOwner[p] != ROW_NONE ? counterOwner[p] : (u32)p;
    EditRec e; e.obj = d.obj[src]; e.opId = d.id[src];
    e.index = elemVisScan[gp] - elemVisScan[objStart[objIdx[p]]];
    if (rowClass[p] == 2) { e.kind = (u32)EK_REMOVE | (ACT_DEL << 16); e.valLen = 0; e.valOff = 0; out[slot[p]] = e; return; }
    const u32 kind = (firstPv[g] == (u32)p && !(firstBare[g] < (u32)p)) ? EK_INSERT : EK_UPDATE;
    e.kind = kind | (flags_action(d.flags[src]) << 16); e.valLen = d.valLen[src]; e.valOff = d.valOff[src];
    if (src != (u32)p) {
      long long total = 0; if (!counter_int64(counterTotal[src], &total)) raise(errWord, KE_COUNTER_RANGE, p);
      e.kind |= EF_COUNTER; e.valLen = (u32)(u64)total; e.valOff = (u32)((u64)total >> 32);
    }
    out[slot[p]] = e;
  }
};
// elemId of an edit = id of the group's insert row (needed for insert edits whose opId differs, i.e. conflicts)
struct EditElemKernel { DocRows d; const u32* rowEmit; const u32* slot; const u32* groupOf; const u32* groupFirst; u64* elemOut; HD void operator()(size_t p) const { if (rowEmit[p]) elemOut[slot[p]] = d.id[groupFirst[groupOf[p]]]; } };

// ---------------------------------------------------------------- incremental list edits: dominance counting
// An item is a query (an op group asking for its list index), a point (a visibility change: weight +1 / -1, or +L for
// a whole typing run) or both at once. tw = time (bits 0..26) | query << 29. The query result is routed by time (every
// group has its own start time). gs / ge = current partition [gs, ge) of the item.
struct DomItem { u32 tw; int w; u32 acc, gs, ge; };
HD u32 dom_tw(u32 time, bool query) { return time | (query ? 1u << 29 : 0u); }
HD u32 dom_time(u32 tw) { return tw & 0x7ffffffu; }
HD bool dom_query(u32 tw) { return (tw >> 29) & 1u; }

// Per-position view of a list element's rows: row p exists from d.time[p] (0 = before this call) and is overwritten at
// minSucc(p) (0 = before this call, 0xffffffff = never). The element whose insert row sits at e owns rows [e, e+rows).
struct ListCtx {
  DocRows d; const u32* succCnt; const u32* newSuccCnt; const u32* firstNewSucc; const u32* groupOf; const u32* groupFirst; const u32* groupRows;
  const u8* arena; const u32* succOff; const u64* succ; const u32* succTime;   // successors of every row with their application times (0 = before this call)
  HD u32 minSucc(u32 p) const { return succCnt[p] > newSuccCnt[p] ? 0u : firstNewSucc[p]; }
  HD long long valueOf(u32 r) const { return counter_operand(arena, d.valLen[r], d.valOff[r]); }
  HD bool isCounterRow(u32 r) const { return flags_action(d.flags[r]) == ACT_SET && (d.valLen[r] & 15) == 8; }
  // Counter row c of the element [e, e + rows) at time T: true if it has increments by then and nothing else overwrote it;
  // *total = summed value (double bits, counter_bits), *lastInc = position of the latest of those increments (new.js:941-966).
  HD bool counterAt(u32 e, u32 rows, u32 c, u32 T, u64* total, u32* lastInc) const {
    u32 last = ROW_NONE;
    for (u32 s = succOff[c]; s < succOff[c + 1]; s++) {
      if (succTime[s] > T) continue;
      u32 q = ROW_NONE;
      for (u32 r = e; r < e + rows; r++) if (d.id[r] == succ[s]) { q = r; break; }
      if (q == ROW_NONE || flags_action(d.flags[q]) != ACT_INC) return false;
      if (last == ROW_NONE || q > last) last = q;
    }
    if (last == ROW_NONE) return false;
    double sum = (double)valueOf(c);
    for (u32 q = c + 1; q <= last; q++) {   // the increments present at T, in row (= opId) order
      bool mine = false; for (u32 s = succOff[c]; s < succOff[c + 1] && !mine; s++) mine = succTime[s] <= T && d.id[q] == succ[s];
      if (mine) sum += (double)valueOf(q);
    }
    *total = counter_bits(sum); *lastInc = last; return true;
  }
  // What the element shows at position q at time T: 1 = the row's own value, 2 = a counter completed by the increment
  // sitting at q (*owner = the counter's row), 0 = nothing
  HD int shownAt(u32 e, u32 rows, u32 q, u32 T, u32* owner, u64* total) const {
    if (d.time[q] > T) return 0;
    const u32 a = flags_action(d.flags[q]);
    if (a == ACT_INC) {
      for (u32 c = e; c < q; c++) {
        if (!isCounterRow(c) || d.time[c] > T) continue;
        bool mine = false; for (u32 s = succOff[c]; s < succOff[c + 1] && !mine; s++) mine = succ[s] == d.id[q];
        if (!mine) continue;
        u32 last; if (counterAt(e, rows, c, T, total, &last) && last == q) { *owner = c; return 2; }
        return 0;
      }
      return 0;
    }
    if (minSucc(q) > T && (a == ACT_SET || (a % 2 == 0 && a != ACT_DEL))) return 1;
    return 0;
  }
  HD bool visAt(u32 e, u32 rows, u32 T) const {   // some row of the element is present and not overwritten after the op at time T
    for (u32 r = e; r < e + rows; r++) if (d.time[r] <= T && minSucc(r) > T) return true;
    return false;
  }
};
// Elements that were visible before the batch are not items: their count in front of a position is one prefix sum.
struct OldVisFlagKernel { ListCtx L; const u32* head; u32* flag; HD void operator()(size_t p) const { flag[p] = (L.d.keyStrLen[p] == NULL32 && head[p] && (L.d.flags[p] & F_INSERT) && L.visAt((u32)p, L.groupRows[L.groupOf[p]], 0)) ? 1u : 0u; } };
// items per position: one merged item for an element with one op group, otherwise its queries first and its points after
// (a query must not see the points of its own element)
// one or two groups on an element: one merged item each, the LATER group first (then neither query can see the other
// group's point: the earlier one fails the time test, the later one the order test); three and more: queries, then points
struct DomItemCountKernel { const u32* nQ; const u32* elemFollower; u32* nItems; HD void operator()(size_t p) const { const u32 k = nQ[p]; nItems[p] = elemFollower[p] ? 0u : (k <= 2 ? k : 2 * k); } };
// Typing runs: consecutive insert ops (consecutive application times) whose elements end up next to each other in the
// document, each touched by nothing else in the batch. Every other query sees such a run entirely or not at all, so the
// run is ONE item: the query of its first op, weighted with the run length; member j has index(head) + j.
struct FollowerFlagKernel {
  MapGroupCtx c; const u32* groupHead; ListCtx L; const u32* gElem; const u32* gT1; const u32* gCount; const u32* nQ; u32* runHeadFlag; u32* elemFollower;
  HD bool plainInsert(size_t t) const {
    const u32 i = c.opAt[t];
    return groupHead[t] && !c.isMapOp(i) && (c.ops.flags[i] & F_INSERT) && gElem[t] != ROW_NONE && nQ[gElem[t]] == 1 && gCount[t] >= 1 && ((gT1[t] >> 29) & 3u) == 2u;
  }
  HD void operator()(size_t t0) const {
    bool f = false;
    if (t0 > 0 && plainInsert(t0) && plainInsert(t0 - 1)) {
      const u32 e = gElem[t0], e1 = gElem[t0 - 1];
      f = e == e1 + L.groupRows[L.groupOf[e1]] && L.d.obj[e] == L.d.obj[e1];
    }
    runHeadFlag[t0] = f ? 0u : 1u;
    if (f) elemFollower[gElem[t0]] = 1;
  }
};
struct RunEndKernel { const u32* runScan; u32* runStart; u32 numOps; HD void operator()(size_t) const { runStart[runScan[numOps]] = numOps; } };   // sentinel behind the last run
struct RunStartKernel { const u32* runHeadFlag; const u32* runScan; u32* runStart; HD void operator()(size_t t) const { if (runHeadFlag[t]) runStart[runScan[t]] = (u32)t; } };
struct DomScanInput {   // per level: low word = 1 if the time bit is clear, high word = the item's weight if the bit is clear
  const u32* tw; const int* w; int bit;
  HD u64 operator()(size_t i) const { return ((tw[i] >> bit) & 1u) == 0 ? (1ull | ((u64)(u32)w[i] << 32)) : 0ull; }
};
struct DomLevelKernel {   // accumulate + stable split of every partition on `bit`; ZW = packed exclusive scan of DomScanInput
  const DomItem* in; DomItem* out; u32* twOut; int* wOut; const u64* ZW; int bit;
  HD void operator()(size_t i) const {
    DomItem it = in[i];
    const u64 s_i = ZW[i], s_gs = ZW[it.gs], s_ge = ZW[it.ge];
    const u32 zg = (u32)s_ge - (u32)s_gs;             // zeros in the partition
    const u32 zb = (u32)s_i - (u32)s_gs;               // zeros before i in the partition
    const bool one = (it.tw >> bit) & 1u;
    u32 dst;
    if (one) {
      if (dom_query(it.tw)) it.acc += (u32)(s_i >> 32) - (u32)(s_gs >> 32);
      dst = it.gs + zg + ((u32)i - it.gs - zb);
      it.gs = it.gs + zg;
    } else {
      dst = it.gs + zb;
      it.ge = it.gs + zg;
    }
    out[dst] = it; twOut[dst] = it.tw; wOut[dst] = it.w;
  }
};
// The last levels in shared memory. After the global levels on the high time bits every partition spans at most
// 2^DOM_LOCAL_BITS distinct times, i.e. at most 2 * 2^DOM_LOCAL_BITS items (one query and one point per time at most), and
// is contiguous: one CTA loads it and runs the remaining levels (same scan + stable split, on shared-memory arrays)
// without touching HBM in between; queries then write their result.
static const int DOM_LOCAL_BITS = 10, DOM_LOCAL_MAX = 2 << DOM_LOCAL_BITS;
struct DomPartHeadKernel { const DomItem* items; u32* flag; HD void operator()(size_t i) const { flag[i] = items[i].gs == (u32)i ? 1u : 0u; } };
struct DomResultKernel {   // route query results back by group start time
  const DomItem* items; u32* qIndex;
  HD void operator()(size_t i) const { if (dom_query(items[i].tw)) qIndex[dom_time(items[i].tw) - 1] = items[i].acc; }
};
// ---------------------------------------------------------------- incremental list edits: one thread per op group
// An op group (new.js:1085-1138) is one insert op, or a run of same-author non-insert ops on one list element that do
// not overwrite each other (GroupSplitKernel). With W = element visible just before the group and V = its rows that are
// visible just after it, updatePatchProperty's state machine (new.js:985-1030) nets out to:
//   V empty: remove if W.   V non-empty, W: update per V row, the first popping earlier edits of the same index
//   (appendUpdate, new.js:798-825).   V non-empty, not W: insert of V[0] then updates.
struct ListGroupKernel {
  int pass; MapGroupCtx c; const u32* groupHead; IdTable t; const u32* rowOfOp; const u32* pos; ListCtx L;
  u32* gCount; u32* gElem; u32* gT1; u32* gQOrd; u32* nQ; u32* elemHasRecs; u32* elemMinT;      // pass 0 out (gT1: T1 | (net weight + 1) << 29 | W << 31)
  const u32* itemBase; const u32* objIdx; const u32* objStart; DomItem* items; u32* twArr; int* wArr; const u32* oldVisScan;   // pass 1: items
  const u32* runHeadFlag; const u32* runScan; const u32* runStart;   // typing runs (FollowerFlagKernel)
  const u32* gBase; const u32* qIndex; EditRec* out; u64* elemOut; u32* objKeyOut; u32* elemPosOut; u32* rowPosOut; u64* errWord;   // pass 2: records
  HD static bool shown(u32 flags) { const u32 a = flags_action(flags); return a == ACT_SET || (a % 2 == 0 && a != ACT_DEL); }
  HD void operator()(size_t t0) const {
    const u32 i0 = c.opAt[t0];
    const bool mine = groupHead[t0] && !c.isMapOp(i0);
    if (pass == 0) {
      u32 n = 0; gElem[t0] = ROW_NONE;
      if (mine) {
        u32 e;
        if (c.ops.flags[i0] & F_INSERT) e = rowOfOp[i0] == ROW_NONE ? ROW_NONE : pos[rowOfOp[i0]];
        else { const u32 row = id_lookup(t, c.ops.key[i0]); e = row == ROW_NONE ? ROW_NONE : L.groupFirst[L.groupOf[pos[row]]]; }
        if (e != ROW_NONE) {
          size_t tl = t0; while (tl + 1 < c.numOps && !groupHead[tl + 1]) tl++;
          const u32 T0 = (u32)t0 + 1, T1 = (u32)tl + 1, rows = L.groupRows[L.groupOf[e]];
          bool W = false; u32 nV = 0;
          for (u32 r = e; r < e + rows; r++) {
            const u32 s = L.d.time[r], x = L.minSucc(r);
            if (s < T0 && x >= T0) W = true;
            u32 owner; u64 total;
            if (L.shownAt(e, rows, r, T1, &owner, &total)) nV++;
          }
          n = nV ? nV : (W ? 1u : 0u);
          const int wNet = (int)L.visAt(e, rows, T1) - (int)L.visAt(e, rows, T0 - 1);
          gElem[t0] = e; gT1[t0] = T1 | ((u32)(wNet + 1) << 29) | (W ? 0x80000000u : 0u);
          if (n || wNet) { gQOrd[t0] = atomic_add(&nQ[e], 1u); atomic_min(&elemMinT[e], T0); } else gQOrd[t0] = ROW_NONE;
          if (nV) elemHasRecs[e] = 1;
        }
      }
      gCount[t0] = n;
      return;
    }
    if (!mine || gElem[t0] == ROW_NONE) return;
    const u32 e = gElem[t0];
    if (pass == 1) {
      if (gQOrd[t0] == ROW_NONE || !runHeadFlag[t0]) return;   // members of a typing run are represented by its head
      int wNet = (int)((gT1[t0] >> 29) & 3u) - 1; const bool isQ = gCount[t0] != 0; const u32 k = nQ[e], o = gQOrd[t0];
      { const u32 run = runScan[t0]; const u32 len = runStart[run + 1] - (u32)t0; if (len > 1) wNet = (int)len; }   // head of a run: all its +1s at once
      DomItem q; q.acc = 0; q.gs = itemBase[objStart[objIdx[e]]]; q.ge = itemBase[objStart[objIdx[e] + 1]];
      if (k <= 2) {
        const u32 at = itemBase[e] + ((k == 2 && elemMinT[e] == (u32)t0 + 1) ? 1u : 0u);   // of two groups the earlier one sits second
        q.tw = dom_tw((u32)t0 + 1, isQ); q.w = wNet; items[at] = q; twArr[at] = q.tw; wArr[at] = q.w;
      } else {
        q.tw = dom_tw((u32)t0 + 1, isQ); q.w = 0; items[itemBase[e] + o] = q; twArr[itemBase[e] + o] = q.tw; wArr[itemBase[e] + o] = 0;
        q.tw = dom_tw((u32)t0 + 1, false); q.w = wNet; items[itemBase[e] + k + o] = q; twArr[itemBase[e] + k + o] = q.tw; wArr[itemBase[e] + k + o] = wNet;
      }
      return;
    }
    if (gCount[t0] == 0) return;
    const u32 T0 = (u32)t0 + 1, T1 = gT1[t0] & 0x1fffffffu; const bool W = gT1[t0] >> 31;
    const u32 runHeadT = runStart[runScan[t0] + runHeadFlag[t0] - 1];   // == t0 unless this op is a member of a typing run
    const u32 rows = L.groupRows[L.groupOf[e]], idx = qIndex[runHeadT] + ((u32)t0 - runHeadT) + oldVisScan[e] - oldVisScan[objStart[objIdx[e]]];
    // Reference quirk, reproduced: when one mergeDocChangeOps call walks from an element straight into the next one
    // (new.js:1116-1121), the insert row of that next element is reported with the list index of the previous element:
    // listIndex is only advanced after updatePatchProperty has seen the row (new.js:1204-1211). It matters for the edits
    // that row itself produces (its own value, or the remove of an element whose insert row was the visible one).
    u32 headIdx = idx;
    if (t0 > 0 && !(c.ops.flags[i0] & F_INSERT)) {
      size_t tp = t0 - 1; while (tp > 0 && !groupHead[tp]) tp--;
      const u32 ip = c.opAt[tp];
      if (!c.isMapOp(ip) && !(c.ops.flags[ip] & F_INSERT) && c.samePass(ip, i0) && id_actor(c.ops.id[ip]) == id_actor(c.ops.id[i0]) && c.ops.obj[ip] == c.ops.obj[i0] && gElem[tp] != ROW_NONE && gElem[tp] < e &&
          L.visAt(gElem[tp], L.groupRows[L.groupOf[gElem[tp]]], T0 - 1)) {   // cheap tests first: the walk below can be long
        const u32 e1 = gElem[tp]; u32 p = e;
        while (p > 0 && L.d.obj[p - 1] == L.d.obj[e] && L.d.time[p - 1] >= T0) p--;      // rows that arrive later in this batch were not there yet
        if (p > 0 && L.d.obj[p - 1] == L.d.obj[e] && L.d.keyStrLen[p - 1] == NULL32 && L.groupFirst[L.groupOf[p - 1]] == e1) headIdx = idx - 1;
      }
    }
    u32 k = gBase[t0], nV = 0;
    for (u32 q = e; q < e + rows; q++) {
      u32 owner = 0; u64 total = 0; const int what = L.shownAt(e, rows, q, T1, &owner, &total);
      if (!what) continue;
      const u32 r = what == 2 ? owner : q;
      EditRec rec; rec.obj = L.d.obj[r]; rec.opId = L.d.id[r]; rec.index = q == e ? headIdx : idx; rec.valLen = L.d.valLen[r]; rec.valOff = L.d.valOff[r];
      rec.kind = (nV == 0 ? (W ? (u32)EK_UPDATE | EF_POP : (u32)EK_INSERT) | EF_GROUP_FIRST : (u32)EK_UPDATE) | (flags_action(L.d.flags[r]) << 16);
      if (what == 2) {
        long long v = 0; if (!counter_int64(total, &v)) raise(errWord, KE_COUNTER_RANGE, t0);
        rec.kind |= EF_COUNTER; rec.valLen = (u32)(u64)v; rec.valOff = (u32)((u64)v >> 32);
      }
      out[k] = rec; elemOut[k] = L.d.id[e]; objKeyOut[k] = objIdx[e]; elemPosOut[k] = e; rowPosOut[k] = r; k++; nV++;
    }
    if (nV == 0) {
      const bool atHead = L.d.time[e] < T0 && L.minSucc(e) >= T0;   // the remove is registered at the first previously visible row
      EditRec rec; rec.obj = L.d.obj[e]; rec.opId = c.ops.id[i0]; rec.index = atHead ? headIdx : idx; rec.valLen = 0; rec.valOff = 0; rec.kind = (u32)EK_REMOVE | EF_GROUP_FIRST | (ACT_DEL << 16);
      out[k] = rec; elemOut[k] = 0; objKeyOut[k] = objIdx[e]; elemPosOut[k] = e; rowPosOut[k] = e;
    }
  }
};
// setupPatches link edits on list parents: an update per visible value of the element, at its index after the call
struct ListLinkKernel {
  int pass; ListCtx L; const u32* listLinkTime; const u32* elemVisScan; const u32* objIdx; const u32* objStart; u32* count; const u32* base; u32 recBase;
  EditRec* out; u64* elemOut; u32* objKeyOut; u32* elemPosOut; u32* timeOut; const u32* elemHasLive /* the element already shows in a surviving edit (patchExists, new.js:1472-1476) */;
  HD void operator()(size_t p) const {
    if (listLinkTime[p] == 0xffffffffu || elemHasLive[p]) { if (pass == 0) count[p] = 0; return; }
    const u32 e = (u32)p, rows = L.groupRows[L.groupOf[e]]; u32 n = 0, k = pass ? recBase + base[p] : 0;
    for (u32 r = e; r < e + rows; r++) {
      if (L.succCnt[r] != 0 || !ListGroupKernel::shown(L.d.flags[r])) continue;
      if (pass == 1) {
        EditRec rec; rec.obj = L.d.obj[r]; rec.opId = L.d.id[r]; rec.index = elemVisScan[e] - elemVisScan[objStart[objIdx[e]]]; rec.valLen = L.d.valLen[r]; rec.valOff = L.d.valOff[r];
        rec.kind = (u32)EK_UPDATE | (u32)EF_START | (flags_action(L.d.flags[r]) << 16);   // appended after everything else: never popped, never merged
        out[k] = rec; elemOut[k] = L.d.id[e]; objKeyOut[k] = objIdx[e]; elemPosOut[k] = e; timeOut[k] = 0x80000000u | listLinkTime[p]; k++;
      }
      n++;
    }
    if (pass == 0) count[p] = n;
  }
};
struct GroupTimeKernel { const u32* gBase; const u32* gCount; u32* timeOut; HD void operator()(size_t t0) const { for (u32 k = 0; k < gCount[t0]; k++) timeOut[gBase[t0] + k] = (u32)t0 + 1; } };
// appendUpdate's pops (new.js:798-825) on the ordered record list: the first record of a popping group kills the
// contiguous insert/update records of the same element before it and turns into an insert if one of them was one.
struct EditFixKernel {
  const EditRec* edits; const u32* elemPos; u32* newKind; u32* pred; u32* dead; size_t n;
  HD void operator()(size_t j) const {
    const u32 kind = edits[j].kind; u32 nk = kind & 0xffu; u32 pr = j == 0 ? ROW_NONE : (u32)(j - 1);
    if (kind & EF_POP) {
      bool insertSeen = false; size_t k = j;
      while (k > 0) {
        const EditRec& a = edits[k - 1]; const u32 ka = a.kind & 0xffu;
        if (!(a.obj == edits[j].obj && a.index == edits[j].index && (ka == EK_INSERT || ka == EK_UPDATE))) break;   // by index only, as the reference
        dead[k - 1] = 1; k--;
        if (ka == EK_INSERT) { insertSeen = true; break; }   // an update that an earlier pop turned into an insert had its own insert further down
      }
      if (insertSeen) nk = EK_INSERT;
      pr = k == 0 ? ROW_NONE : (u32)(k - 1);
    }
    newKind[j] = nk; pred[j] = pr;
  }
};
// appendEdit coalescing (new.js:747-782) against the record that was last in the list when this one was appended
struct EditMergeKernel {
  const EditRec* edits; const u64* elem; const u32* newKind; const u32* pred; u32* mergePrev; u32* multi;
  HD u32 cls(const EditRec& r) const { if (r.kind & EF_COUNTER) return 8; const u32 t = r.valLen & 15; return t == 2 ? 1 : t; }   // datatype + typeof of the value (new.js:759-760)
  HD void operator()(size_t j) const {
    bool cont = false; const u32 i = pred[j];
    if (i != ROW_NONE) {
      const EditRec a = edits[i], b = edits[j]; const u32 ka = newKind[i], kb = newKind[j];
      if (a.obj == b.obj) {
        if (ka == EK_INSERT && kb == EK_INSERT) {
          const u32 actA = (a.kind >> 16) & 0xffff, actB = (b.kind >> 16) & 0xffff;
          cont = b.index == a.index + 1 && actA == ACT_SET && actB == ACT_SET && elem[i] == a.opId && elem[j] == b.opId &&
                 id_actor(a.opId) == id_actor(b.opId) && id_ctr(a.opId) + 1 == id_ctr(b.opId) && cls(a) == cls(b);
          if (cont) { multi[i] = 1; multi[j] = 1; }
        } else if (ka == EK_REMOVE && kb == EK_REMOVE) cont = a.index == b.index;
      }
    }
    mergePrev[j] = cont ? 1u : 0u;
  }
};
struct EditLiveKernel {   // also: does any surviving insert carry an elemId different from its opId? (otherwise the elemId section is not shipped)
  const u32* dead; u32* live; const EditRec* edits; const u64* elem; const u32* newKind; u32* needElem; const u32* elemPos; u32* elemHasLive;
  const u32* rowPos; const u32* succCnt; const u32* counterLast;
  HD void operator()(size_t j) const {
    live[j] = dead[j] ? 0u : 1u;
    if (dead[j]) return;
    if (newKind[j] == EK_INSERT && elem[j] != edits[j].opId) *needElem = 1;
    // setupPatches looks for an edit whose opId is one of the element's CURRENT values (new.js:1472-1476)
    if (newKind[j] != EK_REMOVE && (succCnt[rowPos[j]] == 0 || counterLast[rowPos[j]] != ROW_NONE)) elemHasLive[elemPos[j]] = 1;
  }
};
struct EditCompactKernel {
  const EditRec* in; const u64* elemIn; const u32* dead; const u32* slot; const u32* newKind; const u32* mergePrev; const u32* multi; EditRec* out; u64* elemOut; const u32* objKeyIn; u32* objKeyOut;
  HD void operator()(size_t j) const {
    if (dead[j]) return;
    EditRec r = in[j];
    r.kind = newKind[j] | (r.kind & (0xffff0000u | EF_COUNTER)) | (mergePrev[j] ? 0u : (u32)EF_START) | (multi[j] ? (u32)EF_MULTI : 0u);
    out[slot[j]] = r; elemOut[slot[j]] = elemIn[j]; objKeyOut[slot[j]] = objKeyIn[j];
  }
};
// getPatch: runs over the document-ordered edit list (nothing is ever popped there)
struct RunFlagKernel {
  EditRec* edits; const u64* elem; size_t n;
  HD u32 cls(const EditRec& r) const { if (r.kind & EF_COUNTER) return 8; const u32 t = r.valLen & 15; return t == 2 ? 1 : t; }   // datatype + typeof of the value (new.js:759-760)
  HD bool cont(size_t j) const {
    if (j == 0 || j >= n) return false;
    const EditRec a = edits[j - 1], b = edits[j]; const u32 ka = a.kind & 0xff, kb = b.kind & 0xff;
    if (a.obj != b.obj) return false;
    if (ka == EK_INSERT && kb == EK_INSERT) {
      const u32 actA = (a.kind >> 16) & 0xffff, actB = (b.kind >> 16) & 0xffff;
      return b.index == a.index + 1 && actA == ACT_SET && actB == ACT_SET && elem[j - 1] == a.opId && elem[j] == b.opId &&
             id_actor(a.opId) == id_actor(b.opId) && id_ctr(a.opId) + 1 == id_ctr(b.opId) && cls(a) == cls(b);
    }
    return ka == EK_REMOVE && kb == EK_REMOVE && a.index == b.index;
  }
  HD void operator()(size_t j) const {
    u32 f = 0;
    const bool c0 = cont(j);
    if (!c0) f |= EF_START;
    if ((edits[j].kind & 0xff) == EK_INSERT && (c0 || cont(j + 1))) f |= EF_MULTI;
    atomic_or(&edits[j].kind, f);
  }
};

}  // namespace amg
