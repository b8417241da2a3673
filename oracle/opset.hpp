// ORACLE — TEST INFRASTRUCTURE ONLY (see codec.hpp header).
// CPU restatement of automerge-classic's op-set engine (class BackendDoc), sequential, one
// applyOps() call at a time, with the reference's <=600-op block structure, Bloom filters and block
// metadata, so that it can be pinned on the reference's own byte-exact tests
// (test/new_backend_test.js checkColumns blocks) before it is trusted as the parity checker.
//
// Difference in representation (not in behaviour): the reference keeps every block as encoded
// columns and re-decodes / re-encodes one block per applyOps call; this restatement keeps blocks as
// decoded rows and encodes columns on demand (blockColumns()), which yields the same canonical bytes.
//
// Follows (reference paths relative to /root/reference), function by function:
//   backend/new.js:50-192    seekWithinBlock          backend/new.js:199-216   visibleListElements
//   backend/new.js:227-317   seekToOp                 backend/new.js:329-364   bloomFilterAdd/Contains
//   backend/new.js:370-421   updateBlockMetadata      backend/new.js:426-459   addBlockOperation
//   backend/new.js:465-491   splitBlock               backend/new.js:570-610   readOperation
//   backend/new.js:658-724   readNextDocOp / readNextChangeOp
//   backend/new.js:747-869   appendEdit / appendUpdate / convertInsertToUpdate
//   backend/new.js:884-1040  updatePatchProperty      backend/new.js:1052-1290 mergeDocChangeOps
//   backend/new.js:1304-1380 applyOps                 backend/new.js:1387-1451 updateBlockColumns / getActorTable
//   backend/new.js:1461-1528 setupPatches             backend/new.js:1550-1597 applyChanges (causal gate)
//   backend/new.js:1604-1635 documentPatch            backend/new.js:1645-1692 readDocumentChanges / appendChange
//   backend/new.js:1694-2069 class BackendDoc
#pragma once
#include <memory>
#include <set>
#include <unordered_map>
#include "columnar.hpp"

namespace orc {

static const int MAX_BLOCK_SIZE = 600;
static const int BLOOM_BITS_PER_ENTRY = 10, BLOOM_NUM_PROBES = 7;
static const int BLOOM_FILTER_SIZE = BLOOM_BITS_PER_ENTRY * MAX_BLOCK_SIZE / 8;

static const int64_t NUL = -1;     // JS null for numeric cells
static const int64_t UNDEF = -2;   // JS undefined for block metadata

// A generic cell of an unknown column (new.js:570-610 readOperation keeps them verbatim)
struct Cell {
  enum K { C_NULL, C_NUM, C_STR, C_BYTES, C_LIST } k = C_NULL;
  int64_t num = 0; std::string str; std::vector<RV> list;
};

// One operation row. Change ops carry preds in succ*, document ops carry succs.
struct Op {
  int64_t objActor = NUL, objCtr = NUL, keyActor = NUL, keyCtr = NUL;
  bool hasKeyStr = false; std::string keyStr;
  int64_t idActor = NUL, idCtr = NUL; bool insert = false;
  int64_t action = NUL, valLen = NUL; std::string valRaw;
  int64_t chldActor = NUL, chldCtr = NUL;
  std::vector<int64_t> succActor, succCtr;             // succ (doc op) or pred (change op)
  std::vector<std::pair<int, Cell>> extra;             // unknown columns (columnId, cell)
  int64_t succNum() const { return (int64_t)succCtr.size(); }
};

template <class K, class V> struct OMap {   // insertion-ordered map (JS object with non-integer keys)
  std::vector<std::pair<K, V>> items;
  V* find(const K& k) { for (auto& it : items) if (it.first == k) return &it.second; return nullptr; }
  const V* find(const K& k) const { for (auto& it : items) if (it.first == k) return &it.second; return nullptr; }
  V& operator[](const K& k) { if (V* v = find(k)) return *v; items.emplace_back(k, V()); return items.back().second; }
  void set(const K& k, V v) { if (V* p = find(k)) *p = std::move(v); else items.emplace_back(k, std::move(v)); }
  void erase(const K& k) { for (size_t i = 0; i < items.size(); i++) if (items[i].first == k) { items.erase(items.begin() + i); return; } }
  size_t size() const { return items.size(); }
  bool empty() const { return items.empty(); }
};

struct PObj;
struct PVal {   // a value in a patch: primitive {type:'value',...} or (a reference to) an object patch
  std::shared_ptr<PObj> obj; Prim prim;
  bool isObj() const { return (bool)obj; }
};
struct Edit {
  enum A { INSERT, MULTI_INSERT, UPDATE, REMOVE } action = INSERT;
  int64_t index = 0, count = 0; std::string elemId, opId; bool hasOpId = false;
  PVal value; std::vector<Prim> values; std::string datatype; int datatypeNum = -1; bool hasDatatype = false;
};
struct PObj {
  std::string objectId, type; bool typeNull = false;     // type null for unknown make* actions
  OMap<std::string, OMap<std::string, PVal>> props; std::vector<Edit> edits;
  bool isList() const { return type == "list" || type == "text"; }
};
typedef std::shared_ptr<PObj> PObjP;
typedef std::map<std::string, PObjP> Patches;

struct ChildVal { bool isObj = false; std::string objectId, type; bool typeNull = false; Prim prim; };
struct ObjMeta {
  std::string parentObj; bool hasParent = false; std::string parentKey, opId, type; bool typeNull = false;
  OMap<std::string, OMap<std::string, ChildVal>> children;
};

struct Block {
  std::vector<Op> ops;
  uint8_t bloom[BLOOM_FILTER_SIZE];
  int64_t numOps = 0; bool hasLastKey = false; std::string lastKey;
  int64_t numVisible = UNDEF, lastObjectActor = UNDEF, lastObjectCtr = UNDEF;
  int64_t firstVisibleActor = UNDEF, firstVisibleCtr = UNDEF, lastVisibleActor = UNDEF, lastVisibleCtr = UNDEF;
  Block() { memset(bloom, 0, sizeof(bloom)); }
};
typedef std::shared_ptr<Block> BlockP;

static inline const char* objectTypeOf(int64_t action, bool& isNull) {
  isNull = false;
  switch (action) { case A_MAKE_MAP: return "map"; case A_MAKE_LIST: return "list"; case A_MAKE_TEXT: return "text"; case A_MAKE_TABLE: return "table"; }
  isNull = true; return "";
}
static inline PObjP emptyObjectPatch(const std::string& objectId, const std::string& type, bool typeNull) {
  auto p = std::make_shared<PObj>(); p->objectId = objectId; p->type = type; p->typeNull = typeNull; return p;
}

// new.js:329-364
static inline void bloomFilterAdd(uint8_t* bloom, int64_t elemIdActor, int64_t elemIdCtr) {
  const int64_t modulo = 8 * BLOOM_FILTER_SIZE; int64_t x = elemIdCtr % modulo, y = elemIdActor % modulo;
  int64_t z = (int64_t)((uint32_t)((uint64_t)(uint32_t)((int32_t)elemIdCtr ^ (int32_t)elemIdActor) * 16777619ULL)) % modulo;
  // (ids decoded from a corrupt document can be negative; a Uint8Array ignores a store at a negative index, new.js:329-345)
  for (int i = 0; i < BLOOM_NUM_PROBES; i++) { if (x >= 0) bloom[x >> 3] |= 1 << (x & 7); x = (x + y) % modulo; y = (y + z) % modulo; }
}
static inline bool bloomFilterContains(const uint8_t* bloom, int64_t elemIdActor, int64_t elemIdCtr) {
  const int64_t modulo = 8 * BLOOM_FILTER_SIZE; int64_t x = elemIdCtr % modulo, y = elemIdActor % modulo;
  int64_t z = (int64_t)((uint32_t)((uint64_t)(uint32_t)((int32_t)elemIdCtr ^ (int32_t)elemIdActor) * 16777619ULL)) % modulo;
  for (int i = 0; i < BLOOM_NUM_PROBES; i++) { if (x < 0 || (bloom[x >> 3] & (1 << (x & 7))) == 0) return false; x = (x + y) % modulo; y = (y + z) % modulo; }   // (a load at a negative index is undefined -> 0)
  return true;
}

struct DocState {
  int64_t maxOp = 0;
  std::vector<std::string> actorIds;
  std::vector<std::string> heads;
  std::map<std::string, int64_t> clock;
  std::vector<BlockP> blocks;
  std::map<std::string, ObjMeta> objectMeta;
  std::vector<int> extraColumnIds;   // unknown column ids present in the doc (sorted)
  std::unordered_map<std::string, int64_t>* changeIndexByHash = nullptr;
  const std::string& actorOf(int64_t n) const { static const std::string undef = "undefined"; return (n >= 0 && n < (int64_t)actorIds.size()) ? actorIds[n] : undef; }
  // actorIds.indexOf(a): the first index holding a, or -1. A DocState only appends to actorIds after filling it, so the
  // index map is extended with the new entries; it is rebuilt if the vector shrank. (A linear scan per change made a call
  // that brings tens of thousands of new actors quadratic.)
  int64_t indexOfActor(const std::string& a) const {
    if (actorIndexed > actorIds.size()) { actorIndex.clear(); actorIndexed = 0; }
    for (; actorIndexed < actorIds.size(); actorIndexed++) actorIndex.emplace(actorIds[actorIndexed], (int64_t)actorIndexed);
    auto it = actorIndex.find(a);
    if (it != actorIndex.end() && actorIds[it->second] == a) return it->second;
    if (it == actorIndex.end()) return -1;
    for (size_t i = 0; i < actorIds.size(); i++) if (actorIds[i] == a) return (int64_t)i;   // the vector was rewritten in place
    return -1;
  }
  mutable std::unordered_map<std::string, int64_t> actorIndex;
  mutable size_t actorIndexed = 0;
};

struct SeekOps {   // the `ops` argument of seekToOp / seekWithinBlock (new.js:1308-1312)
  bool objNull = true; std::string objActor; int64_t objActorNum = NUL, objCtr = NUL;
  bool keyActorNull = true; std::string keyActor; int64_t keyActorNum = NUL, keyCtr = NUL;
  bool hasKeyStr = false; std::string keyStr;
  std::string idActor; int64_t idCtr = NUL; bool insert = false;
};
struct SeekResult { bool found; int64_t skipCount, visibleCount; };

// JS value that is null, undefined or a string (an actorId looked up through actorIds[...])
struct JStr { int kind = 0; /* 0 null, 1 undefined, 2 string */ std::string s; };

// new.js:50-192. The reference's column decoders are replaced by cursors over decoded rows; a read
// past the end of a block yields null / false / undefined exactly as the reference's decoders do.
// NB the object cursor (objCtrD/objActorD) and the key / id cursors advance independently, as in
// the reference (after the object seek the object cursor is one row ahead of skipCount).
static SeekResult seekWithinBlock(const SeekOps& ops, const Block& blk, const DocState& ds, bool resumeInsertion) {
  const std::vector<Op>& rows = blk.ops; const int64_t n = (int64_t)rows.size();
  int64_t skipCount = 0, visibleCount = 0; bool elemVisible = false;
  bool nObjCtrNull = true; int64_t nObjCtr = NUL; JStr nObjActor;   // nextObjCtr = null, nextObjActor = null
  int64_t ocur = 0;   // cursor of objCtrD / objActorD / actionD
  auto readObjViaTable = [&]() {   // nextObjCtr = objCtrD.readValue(); nextObjActor = actorIds[objActorD.readValue()]
    if (ocur < n) {
      nObjCtrNull = rows[ocur].objCtr == NUL; nObjCtr = rows[ocur].objCtr;
      if (rows[ocur].objActor == NUL || rows[ocur].objActor >= (int64_t)ds.actorIds.size()) nObjActor.kind = 1;
      else { nObjActor.kind = 2; nObjActor.s = ds.actorIds[rows[ocur].objActor]; }
    } else { nObjCtrNull = true; nObjActor.kind = 1; }
    ocur++;
  };
  auto objEq = [&]() -> bool {   // nextObjCtr === objCtr && nextObjActor === objActor
    if (ops.objNull) return nObjCtrNull && nObjActor.kind == 0;
    return !nObjCtrNull && nObjCtr == ops.objCtr && nObjActor.kind == 2 && nObjActor.s == ops.objActor;
  };

  // Seek to the beginning of the object being updated
  if (!ops.objNull && !resumeInsertion) {
    while (ocur < n) {
      readObjViaTable();
      if (nObjCtrNull || nObjActor.kind != 2 || nObjCtr < ops.objCtr || (nObjCtr == ops.objCtr && nObjActor.s < ops.objActor)) skipCount += 1;
      else break;
    }
  }
  if (!objEq() && !resumeInsertion) return {true, skipCount, visibleCount};

  // Seek to the appropriate key (if string key is used)
  if (ops.hasKeyStr) {
    int64_t kcur = skipCount;   // keyStrD.skipValues(skipCount)
    bool keyColEmpty = true; for (auto& r : rows) if (r.hasKeyStr) { keyColEmpty = false; break; }
    while (!keyColEmpty && kcur < n) {
      // objActorIndex = objActorD.readValue(); nextObjActor = index === null ? null : actorIds[index]
      if (ocur < n) {
        const Op& o = rows[ocur];
        if (o.objActor == NUL) nObjActor.kind = 0;
        else if (o.objActor >= (int64_t)ds.actorIds.size()) nObjActor.kind = 1;
        else { nObjActor.kind = 2; nObjActor.s = ds.actorIds[o.objActor]; }
        nObjCtrNull = o.objCtr == NUL; nObjCtr = o.objCtr;
      } else { nObjActor.kind = 0; nObjCtrNull = true; }
      ocur++;
      const Op& r = rows[kcur]; kcur++;
      if (r.hasKeyStr && js_less(r.keyStr, ops.keyStr) && objEq()) skipCount += 1; else break;
    }
    return {true, skipCount, visibleCount};
  }

  int64_t icur = skipCount;   // idCtrD/idActorD/insertD/succNumD.skipValues(skipCount)
  bool nIdNull = true; int64_t nIdCtr = NUL; JStr nIdActor; bool nInsert = false; bool nSuccNull = true; int64_t nSuccNum = 0;
  auto readId = [&]() {
    if (icur < n) {
      const Op& r = rows[icur]; nIdNull = false; nIdCtr = r.idCtr; nInsert = r.insert; nSuccNull = false; nSuccNum = r.succNum();
      if (r.idActor == NUL || r.idActor >= (int64_t)ds.actorIds.size()) nIdActor.kind = 1; else { nIdActor.kind = 2; nIdActor.s = ds.actorIds[r.idActor]; }
    } else { nIdNull = true; nIdActor.kind = 1; nInsert = false; nSuccNull = true; nSuccNum = 0; }
    icur++;
  };
  auto idDone = [&]() { return icur >= n; };
  auto countVisible = [&]() {
    if (nInsert) elemVisible = false;
    if (!nSuccNull && nSuccNum == 0 && !elemVisible) { visibleCount += 1; elemVisible = true; }
  };
  auto idEqKey = [&]() { return !nIdNull && nIdCtr == ops.keyCtr && nIdActor.kind == 2 && !ops.keyActorNull && nIdActor.s == ops.keyActor; };
  readId();

  if (ops.insert) {
    // If insertion is not at the head, search for the reference element
    if (!resumeInsertion && ops.keyCtr != NUL && ops.keyCtr > 0 && !ops.keyActorNull) {
      skipCount += 1;
      while (!idDone() && !idEqKey()) {
        countVisible();
        readId(); readObjViaTable();
        if (objEq()) skipCount += 1; else break;
      }
      if (!objEq() || !idEqKey() || !nInsert) return {false, skipCount, visibleCount};
      countVisible();
      // Set up the next* variables to the operation following the reference element
      if (idDone()) return {true, skipCount, visibleCount};
      readId(); readObjViaTable();
    }
    // Skip over any list elements with greater ID than the new one, and any non-insertions
    while ((!nInsert || (!nIdNull && (nIdCtr > ops.idCtr || (nIdCtr == ops.idCtr && nIdActor.kind == 2 && nIdActor.s > ops.idActor)))) && objEq()) {
      skipCount += 1;
      countVisible();
      if (!idDone()) { readId(); readObjViaTable(); } else break;
    }
  } else if (ops.keyCtr != NUL && ops.keyCtr > 0 && !ops.keyActorNull) {
    // If we are updating an existing list element, seek to just before the referenced ID
    while ((!nInsert || !idEqKey()) && objEq()) {
      skipCount += 1;
      countVisible();
      if (!idDone()) { readId(); readObjViaTable(); } else break;
    }
    if (!objEq() || !idEqKey() || !nInsert) return {false, skipCount, visibleCount};
  }
  return {true, skipCount, visibleCount};
}

// new.js:199-216
static int64_t visibleListElements(const DocState& ds, size_t blockIndex, int64_t objActorNum, int64_t objCtr) {
  const Block& thisBlock = *ds.blocks[blockIndex]; const Block& nextBlock = *ds.blocks[blockIndex + 1];
  if (thisBlock.lastObjectActor != objActorNum || thisBlock.lastObjectCtr != objCtr || thisBlock.numVisible == UNDEF) return 0;
  if (thisBlock.lastVisibleActor == nextBlock.firstVisibleActor && thisBlock.lastVisibleActor != UNDEF &&
      thisBlock.lastVisibleCtr == nextBlock.firstVisibleCtr && thisBlock.lastVisibleCtr != UNDEF) return thisBlock.numVisible - 1;
  return thisBlock.numVisible;
}

struct SeekPos { size_t blockIndex; int64_t skipCount, visibleCount; };

// new.js:227-317
static SeekPos seekToOp(const DocState& ds, const SeekOps& ops) {
  size_t blockIndex = 0; int64_t totalVisible = 0; const size_t nb = ds.blocks.size();
  // Skip any blocks that contain only objects with lower objectIds
  if (!ops.objNull) {
    while (blockIndex < nb - 1) {
      const Block& b = *ds.blocks[blockIndex];
      // blockActor undefined -> comparisons false; blockCtr null -> advance; undefined -> `undefined < x` false
      bool advance = false;
      if (b.lastObjectCtr == NUL) advance = true;
      else if (b.lastObjectCtr != UNDEF) {
        if (b.lastObjectCtr < ops.objCtr) advance = true;
        else if (b.lastObjectCtr == ops.objCtr && b.lastObjectActor >= 0 && b.lastObjectActor < (int64_t)ds.actorIds.size() &&
                 ds.actorIds[b.lastObjectActor] < ops.objActor) advance = true;
      }
      if (advance) blockIndex++; else break;
    }
  }
  if (ops.hasKeyStr) {
    // String key is used. First skip any blocks that contain only lower keys
    while (blockIndex < nb - 1) {
      const Block& b = *ds.blocks[blockIndex];
      if (ops.objCtr == b.lastObjectCtr && ops.objActorNum == b.lastObjectActor && b.hasLastKey && js_less(b.lastKey, ops.keyStr)) blockIndex++; else break;
    }
    SeekResult r = seekWithinBlock(ops, *ds.blocks[blockIndex], ds, false);
    return {blockIndex, r.skipCount, 0};
  }
  // List operation
  const bool insertAtHead = ops.keyCtr == NUL || ops.keyCtr == 0 || ops.keyActorNull;
  const int64_t keyActorNum = ops.keyActorNull ? NUL : ds.indexOfActor(ops.keyActor);
  bool resumeInsertion = false;
  while (true) {
    if (!insertAtHead && !resumeInsertion) {
      while (blockIndex < nb - 1 && ds.blocks[blockIndex]->lastObjectActor == ops.objActorNum &&
             ds.blocks[blockIndex]->lastObjectCtr == ops.objCtr &&
             !bloomFilterContains(ds.blocks[blockIndex]->bloom, keyActorNum < 0 ? 0 : keyActorNum, ops.keyCtr)) {
        if (ds.blocks[blockIndex]->lastObjectCtr > ops.objCtr)
          throw RangeError("Reference element not found: " + std::to_string(ops.keyCtr) + "@" + ops.keyActor);
        totalVisible += visibleListElements(ds, blockIndex, ops.objActorNum, ops.objCtr);
        blockIndex++;
      }
    }
    SeekResult r = seekWithinBlock(ops, *ds.blocks[blockIndex], ds, resumeInsertion);
    if (blockIndex == nb - 1 || ds.blocks[blockIndex]->lastObjectActor != ops.objActorNum || ds.blocks[blockIndex]->lastObjectCtr != ops.objCtr) {
      if (r.found) return {blockIndex, r.skipCount, totalVisible + r.visibleCount};
      throw RangeError("Reference element not found: " + std::to_string(ops.keyCtr) + "@" + ops.keyActor);
    } else if (r.found && r.skipCount < ds.blocks[blockIndex]->numOps) {
      return {blockIndex, r.skipCount, totalVisible + r.visibleCount};
    }
    resumeInsertion = r.found && ops.insert;
    totalVisible += visibleListElements(ds, blockIndex, ops.objActorNum, ops.objCtr);
    blockIndex++;
  }
}

// new.js:370-421
static void updateBlockMetadata(Block& block) {
  memset(block.bloom, 0, sizeof(block.bloom));
  block.numOps = 0; block.hasLastKey = false; block.lastKey.clear(); block.numVisible = UNDEF;
  block.lastObjectActor = UNDEF; block.lastObjectCtr = UNDEF; block.firstVisibleActor = UNDEF; block.firstVisibleCtr = UNDEF;
  block.lastVisibleActor = UNDEF; block.lastVisibleCtr = UNDEF;
  for (const Op& op : block.ops) {
    block.numOps += 1;
    if (block.lastObjectActor != op.objActor || block.lastObjectCtr != op.objCtr) {
      block.numVisible = 0; block.lastObjectActor = op.objActor; block.lastObjectCtr = op.objCtr;
    }
    if (op.hasKeyStr) { block.hasLastKey = true; block.lastKey = op.keyStr; }
    else if (op.insert || op.keyCtr != NUL) {
      block.hasLastKey = false;
      const int64_t elemIdActor = op.insert ? op.idActor : op.keyActor, elemIdCtr = op.insert ? op.idCtr : op.keyCtr;
      bloomFilterAdd(block.bloom, elemIdActor < 0 ? 0 : elemIdActor, elemIdCtr);
      if (op.succNum() == 0) {
        if (block.firstVisibleActor == UNDEF) block.firstVisibleActor = elemIdActor;
        if (block.firstVisibleCtr == UNDEF) block.firstVisibleCtr = elemIdCtr;
        if (block.lastVisibleActor != elemIdActor || block.lastVisibleCtr != elemIdCtr) {
          block.numVisible += 1; block.lastVisibleActor = elemIdActor; block.lastVisibleCtr = elemIdCtr;
        }
      }
    }
  }
}

// new.js:426-459
static void addBlockOperation(Block& block, const Op& op, const DocState& ds, bool isChangeOp) {
  if (op.hasKeyStr) {
    if (block.lastObjectCtr == op.objCtr && block.lastObjectActor == op.objActor && (!block.hasLastKey || js_less(block.lastKey, op.keyStr))) {
      block.hasLastKey = true; block.lastKey = op.keyStr;
    }
  } else {
    const int64_t elemIdActor = op.insert ? op.idActor : op.keyActor, elemIdCtr = op.insert ? op.idCtr : op.keyCtr;
    bloomFilterAdd(block.bloom, elemIdActor < 0 ? 0 : elemIdActor, elemIdCtr < 0 ? 0 : elemIdCtr);
    if (op.succNum() == 0 || isChangeOp) {
      if (block.firstVisibleActor == UNDEF) block.firstVisibleActor = elemIdActor;
      if (block.firstVisibleCtr == UNDEF) block.firstVisibleCtr = elemIdCtr;
      block.lastVisibleActor = elemIdActor; block.lastVisibleCtr = elemIdCtr;
    }
  }
  // Keep track of the largest objectId contained within a block
  bool update = false;
  if (block.lastObjectCtr == UNDEF) update = true;
  else if (op.objActor != NUL && op.objCtr != NUL) {
    if (block.lastObjectCtr == NUL || block.lastObjectCtr < op.objCtr) update = true;
    else if (block.lastObjectCtr == op.objCtr && block.lastObjectActor >= 0 && ds.actorOf(block.lastObjectActor) < ds.actorOf(op.objActor)) update = true;
  }
  if (update) {
    block.lastObjectActor = op.objActor; block.lastObjectCtr = op.objCtr;
    block.hasLastKey = op.hasKeyStr; block.lastKey = op.hasKeyStr ? op.keyStr : std::string();
    block.numVisible = 0;
  }
}

// new.js:465-491
static std::vector<BlockP> splitBlock(const Block& block) {
  const int64_t numBlocks = (block.numOps + (int64_t)(0.8 * MAX_BLOCK_SIZE) - 1) / (int64_t)(0.8 * MAX_BLOCK_SIZE);
  std::vector<BlockP> blocks; int64_t opsSoFar = 0;
  for (int64_t i = 1; i <= numBlocks; i++) {
    const int64_t upto = (i * block.numOps + numBlocks - 1) / numBlocks;   // Math.ceil(i * numOps / numBlocks)
    auto nb = std::make_shared<Block>();
    nb->ops.assign(block.ops.begin() + opsSoFar, block.ops.begin() + upto);
    updateBlockMetadata(*nb);
    blocks.push_back(nb); opsSoFar = upto;
  }
  return blocks;
}

// ------------------------------------------------------------------------------------------------
// Column <-> row conversion

struct AnyDecoder {   // columnar.js:539-551 decoderByColumnId
  int columnId; int kind;   // 0 rle-uint, 1 delta, 2 boolean, 3 rle-utf8, 4 raw
  RLEDecoder rle; DeltaDecoder delta; BooleanDecoder boolean; Decoder raw;
  AnyDecoder(int id, const std::string& buf) : columnId(id) {
    switch (id & 7) {
      case INT_DELTA: kind = 1; delta = DeltaDecoder(buf); break;
      case BOOLEAN: kind = 2; boolean = BooleanDecoder(buf); break;
      case STRING_RLE: kind = 3; rle = RLEDecoder(T_UTF8, buf); break;
      case VALUE_RAW: kind = 4; raw = Decoder(buf); break;
      default: kind = 0; rle = RLEDecoder(T_UINT, buf); break;
    }
  }
  bool done() const { switch (kind) { case 1: return delta.done(); case 2: return boolean.done(); case 4: return raw.done(); default: return rle.done(); } }
  RV readValue() {
    switch (kind) { case 1: return delta.readValue(); case 2: return RV::Num(boolean.readValue() ? 1 : 0); default: return rle.readValue(); }
  }
};

// Reads all rows out of a set of columns (new.js:570-610 readOperation applied until the action
// column is exhausted). `predOrSucc` group id is 7 for changes and 8 for documents.
static std::vector<Op> readAllOps(const std::vector<Column>& columns, const int* spec, size_t specLen, int groupId,
                                  const std::vector<int64_t>* actorTable, bool untilAllDone = false) {
  static const std::string empty;
  // makeDecoders (columnar.js:553-575): merge the known column spec with the columns present
  std::vector<int> ids;
  { size_t ci = 0, si = 0;
    while (ci < columns.size() || si < specLen) {
      if (ci == columns.size() || (si < specLen && spec[si] < columns[ci].columnId)) ids.push_back(spec[si++]);
      else if (si == specLen || columns[ci].columnId < spec[si]) ids.push_back(columns[ci++].columnId);
      else { ids.push_back(spec[si]); ci++; si++; }
    } }
  std::vector<AnyDecoder> decs; decs.reserve(ids.size());
  for (int id : ids) {
    const std::string* buf = &empty; for (auto& c : columns) if (c.columnId == id) buf = &c.buffer;
    decs.emplace_back(id, *buf);
  }
  int actionIx = -1; for (size_t i = 0; i < ids.size(); i++) if (ids[i] == COL_ACTION) actionIx = (int)i;
  std::vector<Op> ops;
  auto mapActor = [&](const RV& v) -> int64_t {
    if (v.null) return NUL;
    if (!actorTable) return v.num;
    if (v.num < 0 || v.num >= (int64_t)actorTable->size()) throw RangeError("actor index out of range: " + std::to_string(v.num));
    return (*actorTable)[v.num];
  };
  while (true) {
    if (untilAllDone) { bool any = false; for (auto& d : decs) if (!d.done()) any = true; if (!any) break; }
    else if (decs[actionIx].done()) break;
    Op op; int lastGroup = -1; int64_t lastCard = 0; int valueColumn = -1; int64_t valueBytes = 0;
    std::vector<RV> grpActor, grpCtr;
    for (auto& d : decs) {
      const int id = d.columnId, type = id & 7, group = id >> 4;
      const bool known = std::find(spec, spec + specLen, id) != spec + specLen;
      if (type == VALUE_RAW) {
        if (id != valueColumn) throw RangeError("unexpected VALUE_RAW column");
        std::string bytes = d.raw.readRawBytes((size_t)valueBytes);
        if (id == COL_VAL_RAW) op.valRaw = bytes; else { Cell c; c.k = Cell::C_BYTES; c.str = bytes; op.extra.emplace_back(id, c); }
      } else if (type == GROUP_CARD) {
        lastGroup = group; RV v = d.readValue(); lastCard = v.null ? 0 : v.num;
        if (!(known && group == groupId)) { Cell c; c.k = Cell::C_NUM; c.num = lastCard; op.extra.emplace_back(id, c); }
      } else if (group == lastGroup) {
        std::vector<RV> vals;
        if (type == VALUE_LEN) { valueColumn = id + 1; valueBytes = 0; }
        for (int64_t i = 0; i < lastCard; i++) {
          RV v = d.readValue();
          if (type == ACTOR_ID && actorTable && !v.null) v = RV::Num(mapActor(v));
          vals.push_back(v);
        }
        if (known && group == groupId && type == ACTOR_ID) grpActor = vals;
        else if (known && group == groupId && type == INT_DELTA) grpCtr = vals;
        else { Cell c; c.k = Cell::C_LIST; c.list = vals; op.extra.emplace_back(id, c); }
      } else {
        RV v = d.readValue();
        if (type == ACTOR_ID && actorTable && !v.null) v = RV::Num(mapActor(v));
        if (type == VALUE_LEN) { valueColumn = id + 1; valueBytes = v.null ? 0 : (int64_t)((uint64_t)v.num >> 4); }
        auto num = [&]() { return v.null ? NUL : v.num; };
        switch (known ? id : -1) {
          case COL_OBJ_ACTOR: op.objActor = num(); break;   case COL_OBJ_CTR: op.objCtr = num(); break;
          case COL_KEY_ACTOR: op.keyActor = num(); break;   case COL_KEY_CTR: op.keyCtr = num(); break;
          case COL_KEY_STR: op.hasKeyStr = !v.null; op.keyStr = v.str; break;
          case COL_ID_ACTOR: op.idActor = num(); break;     case COL_ID_CTR: op.idCtr = num(); break;
          case COL_INSERT: op.insert = !v.null && v.num != 0; break;
          case COL_ACTION: op.action = num(); break;        case COL_VAL_LEN: op.valLen = num(); break;
          case COL_CHLD_ACTOR: op.chldActor = num(); break; case COL_CHLD_CTR: op.chldCtr = num(); break;
          default: { Cell c; if (v.null) c.k = Cell::C_NULL; else if (v.isStr) { c.k = Cell::C_STR; c.str = v.str; } else { c.k = Cell::C_NUM; c.num = v.num; }
                     op.extra.emplace_back(id, c); }
        }
      }
    }
    for (size_t i = 0; i < grpCtr.size() || i < grpActor.size(); i++) {
      op.succActor.push_back(i < grpActor.size() && !grpActor[i].null ? grpActor[i].num : NUL);
      op.succCtr.push_back(i < grpCtr.size() && !grpCtr[i].null ? grpCtr[i].num : NUL);
    }
    ops.push_back(std::move(op));
  }
  return ops;
}

// Encodes rows as document op columns (the inverse of readAllOps with DOC_OPS_COLUMN_IDS); follows
// appendOperation (new.js:617-650) with encoderByColumnId (columnar.js:525-537). `allIds` lists the
// doc's column ids (known + unknown, ascending).
static std::vector<Column> encodeDocOps(const std::vector<Op>& ops, const std::vector<int>& extraIds) {
  std::vector<int> ids(std::begin(DOC_OPS_COLUMN_IDS), std::end(DOC_OPS_COLUMN_IDS));
  for (int id : extraIds) ids.push_back(id);
  std::sort(ids.begin(), ids.end());
  std::vector<Column> out;
  for (int id : ids) {
    const int type = id & 7; Column col{id, std::string()};
    const bool known = std::find(std::begin(DOC_OPS_COLUMN_IDS), std::end(DOC_OPS_COLUMN_IDS), id) != std::end(DOC_OPS_COLUMN_IDS);
    auto extraOf = [&](const Op& op) -> const Cell* { for (auto& e : op.extra) if (e.first == id) return &e.second; return nullptr; };
    auto N = [](int64_t v) { return v == NUL ? RV() : RV::Num(v); };
    if (type == BOOLEAN) {
      BooleanEncoder e;
      for (auto& op : ops) { if (id == COL_INSERT) e.appendValue(op.insert); else { const Cell* c = extraOf(op); e.appendValue(c && c->k == Cell::C_NUM && c->num != 0); } }
      col.buffer = e.finish();
    } else if (type == VALUE_RAW) {
      for (auto& op : ops) { if (id == COL_VAL_RAW) col.buffer += op.valRaw; else if (const Cell* c = extraOf(op)) col.buffer += c->str; }
    } else {
      std::unique_ptr<RLEEncoder> e;
      if (type == INT_DELTA) e.reset(new DeltaEncoder()); else if (type == STRING_RLE) e.reset(new RLEEncoder(T_UTF8)); else e.reset(new RLEEncoder(T_UINT));
      int groupCardId = (id >> 4) << 4;   // the GROUP_CARD column of this column's group, if any
      for (auto& op : ops) {
        if (!known) {
          const Cell* c = extraOf(op);
          if (type == GROUP_CARD) e->appendValue(RV::Num(c ? c->num : 0));
          else if (c && c->k == Cell::C_LIST) { for (auto& v : c->list) e->appendValue(v); }
          else if (c && c->k == Cell::C_NUM) e->appendValue(RV::Num(c->num));
          else if (c && c->k == Cell::C_STR) e->appendValue(RV::Str(c->str));
          else {
            // blank value: group members get `cardinality` blanks, VALUE_LEN blank is 0 (new.js:642-647)
            const Cell* card = nullptr; for (auto& x : op.extra) if (x.first == groupCardId && groupCardId != id) card = &x.second;
            int64_t count = card ? card->num : 1; if (card == nullptr && false) count = 1;
            bool inGroup = false; for (int other : ids) if (other == groupCardId && (other & 7) == GROUP_CARD && other != id) inGroup = true;
            if (inGroup && !card) count = 0;
            e->appendValue(type == VALUE_LEN ? RV::Num(0) : RV(), count);
          }
          continue;
        }
        switch (id) {
          case COL_OBJ_ACTOR: e->appendValue(N(op.objActor)); break;   case COL_OBJ_CTR: e->appendValue(N(op.objCtr)); break;
          case COL_KEY_ACTOR: e->appendValue(N(op.keyActor)); break;   case COL_KEY_CTR: e->appendValue(N(op.keyCtr)); break;
          case COL_KEY_STR: e->appendValue(op.hasKeyStr ? RV::Str(op.keyStr) : RV()); break;
          case COL_ID_ACTOR: e->appendValue(N(op.idActor)); break;     case COL_ID_CTR: e->appendValue(N(op.idCtr)); break;
          case COL_ACTION: e->appendValue(N(op.action)); break;        case COL_VAL_LEN: e->appendValue(N(op.valLen)); break;
          case COL_CHLD_ACTOR: e->appendValue(N(op.chldActor)); break; case COL_CHLD_CTR: e->appendValue(N(op.chldCtr)); break;
          case COL_SUCC_NUM: e->appendValue(RV::Num(op.succNum())); break;
          case COL_SUCC_ACTOR: for (auto v : op.succActor) e->appendValue(N(v)); break;
          case COL_SUCC_CTR: for (auto v : op.succCtr) e->appendValue(N(v)); break;
        }
      }
      col.buffer = e->finish();
    }
    out.push_back(std::move(col));
  }
  return out;
}

}  // namespace orc
