// amgpu — kernels #3: op-set apply as global sort / rank / scan passes over the whole op table.
//
// Replaces the reference's one-op-at-a-time block rewriting (paths relative to /root/reference):
//   backend/new.js:227-317, 50-192   seekToOp / seekWithinBlock (position search; RGA skip rule :145-163)
//   backend/new.js:1052-1290         mergeDocChangeOps (pred -> succ, opId ordering among same-key ops)
//   backend/new.js:1304-1380         applyOps (block rewrite)
// Document order (SURVEY.md Appendix B): objects by (ctr, actorId string), map rows by key (UTF-16
// order) then opId, list elements in RGA order with the element's update rows after its insert row.
// RGA order equals the pre-order of the insertion tree with siblings in descending opId order,
// provided every insert has a greater counter than its reference element (Lamport property; checked
// in ResolveRowsKernel, KE_LAMPORT otherwise). The pre-order is computed with an Euler tour over
// 4 slots per row and Wyllie pointer jumping, log2(n) passes (ListRankInPlaceKernel on the device, ListRankPackedKernel in
// the emulation build).
#pragma once
#include "gate.cuh"

namespace amg {

static const u32 ROW_NONE = 0xffffffffu;   // no row: _root object / _head element / not found
static const u32 ACT_MAKE_MAP = 0, ACT_SET = 1, ACT_MAKE_LIST = 2, ACT_DEL = 3, ACT_MAKE_TEXT = 4, ACT_INC = 5, ACT_MAKE_TABLE = 6, ACT_LINK = 7;

struct DocRows {   // SoA over rows (document rows: every op except `del`)
  u64 *id, *obj, *key; u32 *keyStrOff, *keyStrLen, *flags, *valLen, *valOff, *time;
};

// ordering key of an opId: counter, then rank of the actor's hex string (rb = bits needed for a rank)
struct Ord {
  const u32* actorRank; int rb;
  HD u64 operator()(u64 id) const { return (id_ctr(id) << rb) | (u64)actorRank[id_actor(id)]; }
};

// ---------------------------------------------------------------- new rows: append every non-del op of the batch
struct RowFlagKernel {   // isRow[i] = op i becomes a document row
  const u32* flags; u32* isRow;
  HD void operator()(size_t i) const { isRow[i] = flags_action(flags[i]) != ACT_DEL ? 1u : 0u; }
};
struct AppendRowsKernel {
  OpRows ops; const u32* isRow; const u32* rowSlot /* exclusive scan of isRow */; size_t numOld; DocRows w; u32* rowOfOp;
  HD void operator()(size_t i) const {
    if (!isRow[i]) { rowOfOp[i] = ROW_NONE; return; }
    const size_t r = numOld + rowSlot[i]; rowOfOp[i] = (u32)r;
    w.id[r] = ops.id[i]; w.obj[r] = ops.obj[i]; w.key[r] = ops.key[i]; w.keyStrOff[r] = ops.keyStrOff[i]; w.keyStrLen[r] = ops.keyStrLen[i];
    w.flags[r] = ops.flags[i]; w.valLen[r] = ops.valLen[i]; w.valOff[r] = ops.valOff[i]; w.time[r] = ops.time[i];
  }
};

// ---------------------------------------------------------------- opId -> row table
struct IdTable { u64* keys; u32* vals; u64 mask; };
struct IdInsertKernel {
  const u64* id; IdTable t; u64* errWord;
  HD void operator()(size_t r) const {
    const u64 k = id[r]; u64 s = mix64(k) & t.mask;
    while (true) {
      const u64 cur = atomic_cas(&t.keys[s], (u64)0, k);
      if (cur == 0) { t.vals[s] = (u32)r; return; }
      if (cur == k) { raise(errWord, KE_DUP_OPID, r); return; }
      s = (s + 1) & t.mask;
    }
  }
};
HD u32 id_lookup(const IdTable& t, u64 k) {
  if (k == 0) return ROW_NONE;
  u64 s = mix64(k) & t.mask;
  while (true) { const u64 cur = t.keys[s]; if (cur == k) return t.vals[s]; if (cur == 0) return ROW_NONE; s = (s + 1) & t.mask; }
}

// ---------------------------------------------------------------- per-row references
struct ResolveRowsKernel {
  DocRows w; IdTable t; Ord ord; size_t numOld;
  u32* objRow; u32* elemRow /* list rows: the element's insert row */; u32* parentRow /* insert rows: reference element row or ROW_NONE (head) */;
  u64* errWord;
  HD void operator()(size_t r) const {
    const u64 obj = w.obj[r]; u32 orow = ROW_NONE;
    if (obj != 0) {
      orow = id_lookup(t, obj);
      // the object of a new op must have been made by a make* op (only those are registered in objectMeta, new.js:904-927: an op in
      // anything else makes the reference fail with a TypeError)
      if (r >= numOld) { const u32 a = orow == ROW_NONE ? 1u : flags_action(w.flags[orow]); if (orow == ROW_NONE || !(a == ACT_MAKE_MAP || a == ACT_MAKE_LIST || a == ACT_MAKE_TEXT || a == ACT_MAKE_TABLE)) raise(errWord, KE_UNSUPPORTED_OP, r); }
    }
    objRow[r] = orow;
    u32 er = ROW_NONE, pr = ROW_NONE;
    if (w.keyStrLen[r] == NULL32) {   // list / text row
      const bool ins = w.flags[r] & F_INSERT; const u64 key = w.key[r];
      if (ins) {
        er = (u32)r;
        if (key != 0) {
          pr = id_lookup(t, key);
          if (pr == ROW_NONE || w.obj[pr] != obj || !(w.flags[pr] & F_INSERT) || w.keyStrLen[pr] != NULL32) { if (r >= numOld) raise(errWord, KE_REF_ELEM, r); pr = ROW_NONE; }
          else if (ord(w.id[pr]) >= ord(w.id[r])) raise(errWord, KE_LAMPORT, r);
        }
      } else {
        er = id_lookup(t, key);
        if (er == ROW_NONE || w.obj[er] != obj || !(w.flags[er] & F_INSERT)) { if (r >= numOld) raise(errWord, KE_REF_ELEM, r); er = ROW_NONE; }
      }
    }
    elemRow[r] = er; parentRow[r] = pr;
  }
};

// ---------------------------------------------------------------- map keys: intern byte strings, rank distinct keys
struct KeySlot { u64 hash; u32 rep; u32 rank; };   // rep = smallest row with this key
struct KeyInternKernel {
  const u8* arena; DocRows w; KeySlot* slots; u64 mask; u32* keySlot;
  HD void operator()(size_t r) const {
    if (w.keyStrLen[r] == NULL32) { keySlot[r] = ROW_NONE; return; }
    u64 h = fnv1a64(arena + w.keyStrOff[r], w.keyStrLen[r]) ^ ((u64)w.keyStrLen[r] << 48); if (h == 0) h = 1;
    u64 s = mix64(h) & mask;
    while (true) {
      const u64 cur = atomic_cas(&slots[s].hash, (u64)0, h);
      if (cur == 0 || cur == h) { atomic_min(&slots[s].rep, (u32)r); keySlot[r] = (u32)s; return; }
      s = (s + 1) & mask;
    }
  }
};
// verifies bytes against the representative (64-bit hash identity) and lists the representatives
struct KeyVerifyKernel {
  const u8* arena; DocRows w; const KeySlot* slots; const u32* keySlot; u32* repList; u32* repCount /* [0] count, [1] max key length */; u64* errWord;
  HD void operator()(size_t r) const {
    const u32 s = keySlot[r]; if (s == ROW_NONE) return;
    const u32 rep = slots[s].rep;
    if (rep == (u32)r) { repList[atomic_add(repCount, 1u)] = (u32)r; atomic_max(repCount + 1, w.keyStrLen[r]); return; }
    const u32 len = w.keyStrLen[r];
    bool same = len == w.keyStrLen[rep];
    for (u32 i = 0; same && i < len; i++) same = arena[w.keyStrOff[r] + i] == arena[w.keyStrOff[rep] + i];
    if (!same) raise(errWord, KE_HASH_COLLISION, r);
  }
};
// 7 bytes of the key at byte position `pos`, transformed so that unsigned compare == UTF-16 code unit
// order (JS string `<`, new.js:84,250,1159): lead bytes EE/EF (U+E000..U+FFFF) sort after F0..F4 (surrogate pairs).
HD u64 key_chunk(const u8* s, u32 len, u32 pos) {
  u64 v = 0; u32 n = 0;
  for (u32 i = 0; i < 7; i++) {
    u32 b = 0;
    if (pos + i < len) { b = s[pos + i]; n++; if (b == 0xEE || b == 0xEF) b += 5; else if (b >= 0xF0 && b <= 0xF4) b -= 2; }
    v = (v << 8) | b;
  }
  return (v << 8) | n;
}
// LSD string sort of the distinct keys: one stable 64-bit sort per 7-byte chunk, last chunk first
struct KeyChunkKernel {
  const u8* arena; DocRows w; const u32* items /* representative rows, current order */; u32 pos; u64* chunk;
  HD void operator()(size_t j) const { const u32 r = items[j]; chunk[j] = key_chunk(arena + w.keyStrOff[r], w.keyStrLen[r], pos); }
};
struct KeyRankKernel {   // after the last pass the position in `items` is the key's rank
  const u32* items; const u32* keySlot; KeySlot* slots;
  HD void operator()(size_t j) const { slots[keySlot[items[j]]].rank = (u32)j; }
};

// ---------------------------------------------------------------- generic helpers
struct IotaKernel { u32* out; HD void operator()(size_t i) const { out[i] = (u32)i; } };
struct FillU32Kernel { u32* out; u32 v; HD void operator()(size_t i) const { out[i] = v; } };
struct FillU64Kernel { u64* out; u64 v; HD void operator()(size_t i) const { out[i] = v; } };
struct GatherU64Kernel { const u64* src; const u32* idx; u64* out; HD void operator()(size_t i) const { out[i] = src[idx[i]]; } };
struct InversePermKernel { const u32* perm; u32* inv; HD void operator()(size_t i) const { inv[perm[i]] = (u32)i; } };
// dense rank from sorted (major, minor) keys: head flag where the key changes
struct HeadFlagKernel { const u64* a; const u64* b; u32* flag; HD void operator()(size_t j) const { flag[j] = (j == 0 || a[j] != a[j - 1] || (b && b[j] != b[j - 1])) ? 1u : 0u; } };

// ---------------------------------------------------------------- RGA order: Euler tour + list ranking
// Compact slots: after the sibling sort the j-th insert row owns 2j (enter) and 2j+1 (exit), so a node's next sibling is
// its memory neighbour; the k-th list object owns 2I+2k (head enter) and 2I+2k+1 (head exit).
struct SiblingKeyKernel {   // sort key (parent code, descending opId) for insert rows; `items` lists the insert rows
  DocRows w; const u32* items; const u32* parentRow; const u32* objRow; Ord ord; int ordBits; u64* key; u64* errWord;
  HD void operator()(size_t j) const {
    const u32 r = items[j]; const u32 pr = parentRow[r];
    if (pr == ROW_NONE && objRow[r] == ROW_NONE) { raise(errWord, KE_UNSUPPORTED_OP, r); key[j] = 0; return; }   // list op on _root
    if (pr == ROW_NONE) { const u32 a = flags_action(w.flags[objRow[r]]); if (a != ACT_MAKE_LIST && a != ACT_MAKE_TEXT) { raise(errWord, KE_UNSUPPORTED_OP, r); key[j] = 0; return; } }   // list op on a map
    const u64 parentCode = pr != ROW_NONE ? ((u64)pr << 1) : (((u64)objRow[r] << 1) | 1);   // head of the object
    const u64 maxOrd = (1ULL << ordBits) - 1;
    key[j] = (parentCode << ordBits) | (maxOrd - ord(w.id[r]));
  }
};
struct ListObjFlagKernel { DocRows w; u32* flag; HD void operator()(size_t r) const { const u32 a = flags_action(w.flags[r]); flag[r] = (a == ACT_MAKE_LIST || a == ACT_MAKE_TEXT) ? 1u : 0u; } };
struct ItemIndexKernel { const u32* items; u32* itemIdx; HD void operator()(size_t j) const { itemIdx[items[j]] = (u32)j; } };
struct EulerLinkKernel {   // after sorting siblings: set first-child and next-sibling links
  const u64* key; int ordBits; const u32* itemIdx; const u32* objSlot; u32* next /* [2I + 2L] */; u32* weight; size_t n;
  HD void operator()(size_t j) const {
    const u64 pc = key[j] >> ordBits;
    const bool firstOfParent = j == 0 || (key[j - 1] >> ordBits) != pc, lastOfParent = j + 1 == n || (key[j + 1] >> ordBits) != pc;
    const u32 parentEnter = (pc & 1) ? (u32)(2 * n + 2 * objSlot[pc >> 1]) : 2 * itemIdx[pc >> 1], parentExit = parentEnter + 1;
    if (firstOfParent) next[parentEnter] = (u32)(2 * j);                      // enter(parent) -> enter(first child)
    next[2 * j + 1] = lastOfParent ? parentExit : (u32)(2 * j + 2);           // exit -> enter(next sibling) | exit(parent)
    weight[2 * j] = 1;
  }
};
struct EulerInitKernel {   // default links: enter -> own exit, exit -> self (terminal until linked)
  u32* next; u32* weight;
  HD void operator()(size_t s) const { next[s] = (s & 1) ? (u32)s : (u32)s + 1; weight[s] = 0; }
};
// Wyllie pointer jumping: rank[s] = sum of weights from s (inclusive) to the end of its list, on (next | rank << 32) packed
// into one word: a jump reads ONE random 8-byte word (one sector) instead of two
// 4-byte words in two arrays (two sectors) - the random reads are what a round costs.
struct ListRankPackKernel { const u32* next; const u32* rank; u64* packed; HD void operator()(size_t s) const { packed[s] = (u64)next[s] | ((u64)rank[s] << 32); } };
struct ListRankPackedKernel {
  const u64* in; u64* out;
  HD void operator()(size_t s) const {
    const u64 me = in[s]; const u32 n = (u32)me;
    if (n == (u32)s) { out[s] = me; return; }
    const u64 nb = in[n];
    out[s] = (u64)(u32)nb | ((u64)((u32)(me >> 32) + (u32)(nb >> 32)) << 32);
  }
};
// The device runs the same jump on one array, in place: a word read while another thread rewrites it is either its old or
// its new (next, weight up to next) pair, both consistent and at least as far along as at the launch's start, so a round
// covers at least what a round over two buffers does, and the last round leaves the same ranks.
struct ListRankInPlaceKernel {
  u64* packed;
  HD void operator()(size_t s) const {
    const u64 me = packed[s]; const u32 n = (u32)me;
    if (n == (u32)s) return;
    const u64 nb = packed[n];
    packed[s] = (u64)(u32)nb | ((u64)((u32)(me >> 32) + (u32)(nb >> 32)) << 32);
  }
};
struct ListRankUnpackKernel { const u64* packed; u32* rank; HD void operator()(size_t s) const { rank[s] = (u32)(packed[s] >> 32); } };
// list position of every list row = number of elements before its element in its object
struct ListPosKernel {
  const u32* rank; const u32* elemRow; const u32* objRow; const u32* itemIdx; const u32* objSlot; u32 numItems; u32* listPos;
  HD void operator()(size_t r) const {
    const u32 e = elemRow[r];
    if (e == ROW_NONE || objRow[e] == ROW_NONE) { listPos[r] = 0; return; }
    listPos[r] = rank[2 * (size_t)numItems + 2 * objSlot[objRow[e]]] - rank[2 * (size_t)itemIdx[e]];   // total(list) - suffix(enter e)
  }
};

// ---------------------------------------------------------------- document order
struct DocKeyKernel {   // field: 0 tertiary (opId within key/element), 1 secondary (key rank / list position), 2 object order
  int field; DocRows w; const u32* perm; const u32* listPos; const KeySlot* keySlots; const u32* keySlot; Ord ord; u64* key;
  HD void operator()(size_t j) const {
    const u32 r = perm[j]; u64 k;
    if (field == 0) k = (w.keyStrLen[r] == NULL32 && (w.flags[r] & F_INSERT)) ? 0 : ord(w.id[r]) + 1;
    else if (field == 1) k = w.keyStrLen[r] == NULL32 ? listPos[r] : keySlots[keySlot[r]].rank;
    else k = w.obj[r] == 0 ? 0 : ord(w.obj[r]) + 1;
    key[j] = k;
  }
};
struct GatherRowsKernel {   // materialise the new document table in document order
  DocRows src, dst; const u32* perm;
  HD void operator()(size_t p) const {
    const u32 r = perm[p];
    dst.id[p] = src.id[r]; dst.obj[p] = src.obj[r]; dst.key[p] = src.key[r]; dst.keyStrOff[p] = src.keyStrOff[r]; dst.keyStrLen[p] = src.keyStrLen[r];
    dst.flags[p] = src.flags[r]; dst.valLen[p] = src.valLen[r]; dst.valOff[p] = src.valOff[r]; dst.time[p] = src.time[r];
  }
};

// ---------------------------------------------------------------- succ lists
// pairs (position of the overwritten row, overwriting opId): old succ entries + one per pred of the batch
struct PredPairsKernel {
  OpRows ops; IdTable t; const u32* pos /* row -> doc position */; const u32* rowOfOp; DocRows w; const u32* elemRow; const u32* keySlot;
  Ord ord; u64* pairKey /* ord of succ */; u32* pairIdx; u64* pairSucc; u32* pairPos; u32* pairTime; size_t pairBase; u64* errWord;
  HD void operator()(size_t i) const {
    const u32 n = ops.predNum[i];
    for (u32 j = 0; j < n; j++) {
      const size_t p = ops.predOff[i] + j; const size_t q = pairBase + p;
      const u32 target = id_lookup(t, ops.predId[p]);
      pairKey[q] = ord(ops.id[i]); pairIdx[q] = (u32)q; pairSucc[q] = ops.id[i]; pairTime[q] = ops.time[i];
      // (an inserting op never meets its preds: the reference places it without looking at the document ops, new.js:1156-1160, 1254-1257)
      if (target == ROW_NONE || (ops.flags[i] & F_INSERT)) { raise(errWord, KE_PRED_MISSING, p); pairPos[q] = 0; continue; }
      // the pred must be an op on the same key / list element of the same object, applied earlier (new.js:1173-1188, 1254-1257)
      // ... and must have the smaller opId (every encoder's startOp exceeds what its author has seen): the reference only looks for
      // a pred among the ops in front of the place the new op takes in opId order (new.js:1172-1187, 1254-1257)
      bool ok = w.obj[target] == ops.obj[i] && w.time[target] < ops.time[i] && ord(ops.predId[p]) < ord(ops.id[i]);
      if (ops.keyStrLen[i] != NULL32) {
        ok = ok && w.keyStrLen[target] != NULL32;
        const u32 r = rowOfOp[i];
        if (ok && r != ROW_NONE) ok = keySlot[r] == keySlot[target];   // a map-key `del` has no row: DelKeyCheckKernel compares bytes
      } else {
        ok = ok && w.keyStrLen[target] == NULL32 && elemRow[target] != ROW_NONE && w.id[elemRow[target]] == ops.key[i];
      }
      if (!ok) raise(errWord, KE_PRED_MISSING, p);
      pairPos[q] = pos[target];
    }
  }
};
// an `inc` op needs a counter to add to: one of its preds must be a `set` of datatype counter (new.js:953-957)
// (its number is decoded when the op is processed, whether or not the counter still shows: decodeValue, new.js:954,
// columnar.js:300-329 - like that of a counter `set`, new.js:944)
struct IncCheckKernel {
  OpRows ops; IdTable t; DocRows w; const u8* arena; u64* errWord;
  HD void operator()(size_t i) const {
    const u32 act = flags_action(ops.flags[i]), tag = ops.valLen[i] & 15;
    if ((act == ACT_INC || (act == ACT_SET && tag == 8)) && (tag == 3 || tag == 4 || tag == 8 || tag == 9)) {
      ByteReader r(arena, ops.valOff[i], ops.valOff[i] + (ops.valLen[i] >> 4));
      if (tag == 3) r.uleb(); else r.sleb();
      if (r.err) raise(errWord, r.err, i);
    }
    if (act != ACT_INC) return;
    if (tag > 4 && tag != 8 && tag != 9) { raise(errWord, KE_UNSUPPORTED_OP, i); return; }   // += of a float / string / bytes value: JavaScript would concatenate or go floating point
    bool ok = false, other = false;
    for (u32 j = 0; j < ops.predNum[i]; j++) {
      const u32 target = id_lookup(t, ops.predId[ops.predOff[i] + j]);
      if (target != ROW_NONE && flags_action(w.flags[target]) == ACT_SET && (w.valLen[target] & 15) == 8) ok = true; else other = true;
    }
    if (!ok) raise(errWord, KE_UNKNOWN_COUNTER, i);
    else if (other) raise(errWord, KE_UNSUPPORTED_OP, i);   // an increment that also overwrites something that is no counter: no encoder writes one
  }
};
// list `del` ops have no row: their element must exist (seekToOp would throw first, new.js:293-301)
struct DelElemCheckKernel {
  OpRows ops; IdTable t; DocRows w; u64* errWord;
  HD void operator()(size_t i) const {
    if (flags_action(ops.flags[i]) != ACT_DEL) return;
    if ((ops.flags[i] & F_INSERT) || ops.predNum[i] == 0) { raise(errWord, KE_UNSUPPORTED_OP, i); return; }   // an inserting `del` (the reference would make a list element of it), a `del` that deletes nothing: no encoder writes one
    if (ops.keyStrLen[i] != NULL32) return;
    const u32 e = id_lookup(t, ops.key[i]);
    if (e == ROW_NONE || w.obj[e] != ops.obj[i] || !(w.flags[e] & F_INSERT) || w.keyStrLen[e] != NULL32) raise(errWord, KE_REF_ELEM, i);
  }
};
// map-key `del` ops have no row: check their preds' keys by bytes
struct DelKeyCheckKernel {
  const u8* arena; OpRows ops; IdTable t; DocRows w; u64* errWord;
  HD void operator()(size_t i) const {
    if (flags_action(ops.flags[i]) != ACT_DEL || ops.keyStrLen[i] == NULL32) return;
    for (u32 j = 0; j < ops.predNum[i]; j++) {
      const u32 target = id_lookup(t, ops.predId[ops.predOff[i] + j]); if (target == ROW_NONE) continue;
      bool same = w.keyStrLen[target] == ops.keyStrLen[i];
      for (u32 k = 0; same && k < ops.keyStrLen[i]; k++) same = arena[w.keyStrOff[target] + k] == arena[ops.keyStrOff[i] + k];
      if (!same) raise(errWord, KE_PRED_MISSING, ops.predOff[i] + j);
    }
  }
};
struct OldPairsKernel {   // old succ entries keep their row; re-key to the row's new position
  const u32* oldSuccOff; const u64* oldSucc; const u32* pos; Ord ord; u64* pairKey; u32* pairIdx; u64* pairSucc; u32* pairPos; u32* pairTime;
  HD void operator()(size_t r) const {
    for (u32 q = oldSuccOff[r]; q < oldSuccOff[r + 1]; q++) { pairKey[q] = ord(oldSucc[q]); pairIdx[q] = q; pairSucc[q] = oldSucc[q]; pairPos[q] = pos[r]; pairTime[q] = 0; }
  }
};
struct CountSuccKernel { const u32* pairPos; u32* cnt; HD void operator()(size_t q) const { atomic_add(&cnt[pairPos[q]], 1u); } };
struct PairPosKeyKernel { const u32* pairPos; const u32* idx; u64* key; HD void operator()(size_t j) const { key[j] = pairPos[idx[j]]; } };
struct WriteSuccKernel {   // pairs are sorted by (position, succ ord): write the CSR payload
  const u32* idx; const u64* pairSucc; u64* succOut; const u32* pairTime; u32* succTimeOut /* application time of the entry, 0 = before this call */;
  HD void operator()(size_t j) const { succOut[j] = pairSucc[idx[j]]; succTimeOut[j] = pairTime[idx[j]]; }
};
// first deleter of each row during this call: min application time over new succ entries
struct FirstSuccTimeKernel {
  const u32* pairPos; const u32* pairTime; u32* firstNewSucc;
  HD void operator()(size_t q) const { if (pairTime[q] != 0) atomic_min(&firstNewSucc[pairPos[q]], pairTime[q]); }
};

}  // namespace amg
