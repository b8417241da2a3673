// ORACLE — TEST INFRASTRUCTURE ONLY (see codec.hpp header).
// Second half of the op-set engine restatement: patch state machine, merge loop, applyOps, causal
// gate and class BackendDoc.  Reference line numbers are given per function (backend/new.js).
#pragma once
#include "opset.hpp"

namespace orc {

static inline std::string opIdStr(int64_t ctr, const std::string& actor) { return std::to_string(ctr) + "@" + actor; }

// new.js:738-741 opIdDelta
static bool opIdDelta(const std::string& id1, const std::string& id2, int64_t delta) {
  size_t a1 = id1.find('@'), a2 = id2.find('@');
  if (a1 == std::string::npos || a2 == std::string::npos) throw RangeError("Not a valid opId: " + (a1 == std::string::npos ? id1 : id2));
  if (id1.compare(a1, std::string::npos, id2, a2, std::string::npos) != 0) return false;
  return std::stoll(id1.substr(0, a1)) + delta == std::stoll(id2.substr(0, a2));
}

// new.js:747-782
static void appendEdit(std::vector<Edit>& edits, Edit next) {
  if (edits.empty()) { edits.push_back(std::move(next)); return; }
  Edit& last = edits.back();
  if (last.action == Edit::INSERT && next.action == Edit::INSERT && last.index == next.index - 1 &&
      !last.value.isObj() && !next.value.isObj() && last.elemId == last.opId && next.elemId == next.opId &&
      opIdDelta(last.elemId, next.elemId, 1) && last.value.prim.sameDatatype(next.value.prim) &&
      last.value.prim.typeOf() == next.value.prim.typeOf()) {
    last.action = Edit::MULTI_INSERT;
    if (!next.value.prim.datatype.empty() || next.value.prim.datatypeNum >= 0) {
      last.hasDatatype = true; last.datatype = next.value.prim.datatype; last.datatypeNum = next.value.prim.datatypeNum;
    }
    last.values = {last.value.prim, next.value.prim};
    last.value = PVal(); last.hasOpId = false; last.opId.clear();
  } else if (last.action == Edit::MULTI_INSERT && next.action == Edit::INSERT &&
             last.index + (int64_t)last.values.size() == next.index && !next.value.isObj() && next.elemId == next.opId &&
             opIdDelta(last.elemId, next.elemId, (int64_t)last.values.size()) &&
             last.datatype == next.value.prim.datatype && last.datatypeNum == next.value.prim.datatypeNum &&
             last.values[0].typeOf() == next.value.prim.typeOf()) {
    last.values.push_back(next.value.prim);
  } else if (last.action == Edit::REMOVE && next.action == Edit::REMOVE && last.index == next.index) {
    last.count += next.count;
  } else {
    edits.push_back(std::move(next));
  }
}

// new.js:798-824
static void appendUpdate(std::vector<Edit>& edits, int64_t index, const std::string& elemId, const std::string& opId, const PVal& value, bool firstUpdate) {
  bool insert = false;
  if (firstUpdate) {
    while (!insert && !edits.empty()) {
      Edit& last = edits.back();
      if ((last.action == Edit::INSERT || last.action == Edit::UPDATE) && last.index == index) {
        insert = (last.action == Edit::INSERT); edits.pop_back();
      } else if (last.action == Edit::MULTI_INSERT && last.index + (int64_t)last.values.size() - 1 == index) {
        last.values.pop_back(); insert = true;
      } else break;
    }
  }
  Edit e; e.index = index; e.opId = opId; e.hasOpId = true; e.value = value;
  if (insert) { e.action = Edit::INSERT; e.elemId = elemId; } else e.action = Edit::UPDATE;
  appendEdit(edits, std::move(e));
}

// new.js:838-869
static void convertInsertToUpdate(std::vector<Edit>& edits, int64_t index, const std::string& elemId) {
  std::vector<Edit> updates;
  while (!edits.empty()) {
    Edit& last = edits.back();
    if (last.action == Edit::INSERT) {
      if (last.index != index) throw RangeError("last edit has unexpected index");
      updates.insert(updates.begin(), last); edits.pop_back(); break;
    } else if (last.action == Edit::UPDATE) {
      if (last.index != index) throw RangeError("last edit has unexpected index");
      updates.insert(updates.begin(), last); edits.pop_back();
    } else throw RangeError("last edit has unexpected action");
  }
  bool firstUpdate = true;
  for (auto& u : updates) { appendUpdate(edits, index, elemId, u.opId, u.value, firstUpdate); firstUpdate = false; }
}

// value is a JavaScript number, as in the reference: `counterState.value += ...` (new.js:944, 958) adds doubles, so a total
// past 2^53 is rounded at each step
struct CounterState { std::string opId; double value = 0; std::set<std::string> succs; };
struct PropState {
  std::vector<Op> visibleOps; bool hasChild = false; int action = 0;   // 0 none, 1 insert, 2 update, 3 remove
  std::map<std::string, std::shared_ptr<CounterState>> counterStates; bool hasCounterStates = false;
};
typedef std::map<std::string, PropState> PropStates;

static PVal primVal(const Op& op) { PVal v; v.prim = decodeValue(op.valLen == NUL ? 0 : op.valLen, op.valRaw); return v; }

// new.js:884-1040
static void updatePatchProperty(Patches& patches, Block* newBlock, const std::string& objectId, const Op& op, DocState& ds,
                                PropStates& propState, int64_t listIndex, bool hasOldSuccNum, int64_t oldSuccNum) {
  const bool isWholeDoc = !newBlock;
  bool typeNull; std::string type = objectTypeOf(op.action, typeNull);   // only used for make* (even) actions
  if (op.action >= NUM_ACTIONS) { typeNull = true; type.clear(); }
  const std::string opId = opIdStr(op.idCtr, ds.actorOf(op.idActor));
  const int64_t elemIdActor = op.insert ? op.idActor : op.keyActor, elemIdCtr = op.insert ? op.idCtr : op.keyCtr;
  const std::string elemId = (op.hasKeyStr && !op.keyStr.empty()) ? op.keyStr : opIdStr(elemIdCtr, ds.actorOf(elemIdActor));
  const bool isMake = op.action != NUL && op.action % 2 == 0;

  if (isMake && !ds.objectMeta.count(opId)) {
    ObjMeta m; m.parentObj = objectId; m.hasParent = true; m.parentKey = elemId; m.opId = opId; m.type = type; m.typeNull = typeNull;
    ds.objectMeta[opId] = m;
    ChildVal cv; cv.isObj = true; cv.objectId = opId; cv.type = type; cv.typeNull = typeNull;
    ds.objectMeta[objectId].children[elemId].set(opId, cv);
  }

  const bool firstOp = !propState.count(elemId);
  PropState& ps = propState[elemId];
  const bool isOverwritten = hasOldSuccNum && op.succNum() > 0;
  if (!isOverwritten) { ps.visibleOps.push_back(op); ps.hasChild = ps.hasChild || isMake; }

  auto metaIt = ds.objectMeta.find(objectId);
  if (metaIt == ds.objectMeta.end()) throw TypeError("Cannot read property 'children' of undefined (unknown object " + objectId + ")");
  const OMap<std::string, ChildVal>* prevChildren = metaIt->second.children.find(elemId);
  if (ps.hasChild || (prevChildren && prevChildren->size() > 0)) {
    OMap<std::string, ChildVal> values;
    for (const Op& visible : ps.visibleOps) {
      const std::string vid = opIdStr(visible.idCtr, ds.actorOf(visible.idActor));
      if (visible.action == A_SET) { ChildVal cv; cv.prim = decodeValue(visible.valLen == NUL ? 0 : visible.valLen, visible.valRaw); values.set(vid, cv); }
      else if (visible.action != NUL && visible.action % 2 == 0) {
        ChildVal cv; cv.isObj = true; cv.objectId = vid; bool tn; cv.type = objectTypeOf(visible.action, tn); cv.typeNull = tn; values.set(vid, cv);
      }
    }
    metaIt->second.children.set(elemId, values);
  }

  bool hasPatch = false; std::string patchKey; PVal patchValue;
  if (isOverwritten && op.action == A_SET && op.valLen != NUL && (op.valLen & 0x0f) == VT_COUNTER) {
    // The initial set operation that creates a counter
    ps.hasCounterStates = true;
    auto cs = std::make_shared<CounterState>(); cs->opId = opId;
    Prim p = decodeValue(op.valLen, op.valRaw); cs->value = p.num();
    for (int64_t i = 0; i < op.succNum(); i++) {
      const std::string succOp = opIdStr(op.succCtr[i], ds.actorOf(op.succActor[i]));
      ps.counterStates[succOp] = cs; cs->succs.insert(succOp);
    }
  } else if (op.action == A_INC) {
    if (!ps.hasCounterStates || !ps.counterStates.count(opId)) throw RangeError("increment operation " + opId + " for unknown counter");
    auto cs = ps.counterStates[opId];
    Prim p = decodeValue(op.valLen == NUL ? 0 : op.valLen, op.valRaw); cs->value += p.k == Prim::P_BOOL ? (p.b ? 1.0 : 0.0) : p.num();
    cs->succs.erase(opId);
    if (cs->succs.empty()) {
      // an integer-valued double in [-2^63, 2^63) is written as that integer, exactly; a larger one as a float
      hasPatch = true; patchKey = cs->opId; patchValue.prim.datatype = "counter";
      if (cs->value >= -9223372036854775808.0 && cs->value < 9223372036854775808.0) { patchValue.prim.k = Prim::P_INT; patchValue.prim.i = (int64_t)cs->value; }
      else { patchValue.prim.k = Prim::P_FLOAT; patchValue.prim.f = cs->value; }
    }
  } else if (!isOverwritten) {
    if (op.action == A_SET) { hasPatch = true; patchKey = opId; patchValue = primVal(op); }
    else if (isMake) {
      if (!patches.count(opId)) patches[opId] = emptyObjectPatch(opId, type, typeNull);
      hasPatch = true; patchKey = opId; patchValue.obj = patches[opId];
    }
  }

  if (!patches.count(objectId)) patches[objectId] = emptyObjectPatch(objectId, metaIt->second.type, metaIt->second.typeNull);
  PObj& patch = *patches[objectId];
  auto adjustVisible = [&](int delta) {
    if (newBlock && newBlock->lastObjectActor == op.objActor && newBlock->lastObjectCtr == op.objCtr) newBlock->numVisible += delta;
  };

  if (!op.hasKeyStr) {
    // Updating a list or text object (with elemId key)
    if (hasOldSuccNum && oldSuccNum == 0 && !isWholeDoc && ps.action == 1) {
      ps.action = 2;
      convertInsertToUpdate(patch.edits, listIndex, elemId);
      adjustVisible(-1);
    }
    if (hasPatch) {
      if (ps.action == 0 && (!hasOldSuccNum || isWholeDoc)) {
        ps.action = 1;
        Edit e; e.action = Edit::INSERT; e.index = listIndex; e.elemId = elemId; e.opId = patchKey; e.hasOpId = true; e.value = patchValue;
        appendEdit(patch.edits, std::move(e));
        adjustVisible(+1);
      } else if (ps.action == 3) {
        if (patch.edits.empty() || patch.edits.back().action != Edit::REMOVE) throw RangeError("last edit has unexpected type");
        if (patch.edits.back().count > 1) patch.edits.back().count -= 1; else patch.edits.pop_back();
        ps.action = 2;
        appendUpdate(patch.edits, listIndex, elemId, patchKey, patchValue, true);
        adjustVisible(+1);
      } else {
        appendUpdate(patch.edits, listIndex, elemId, patchKey, patchValue, ps.action == 0);
        if (ps.action == 0) ps.action = 2;
      }
    } else if (hasOldSuccNum && oldSuccNum == 0 && ps.action == 0) {
      ps.action = 3;
      Edit e; e.action = Edit::REMOVE; e.index = listIndex; e.count = 1;
      appendEdit(patch.edits, std::move(e));
      adjustVisible(-1);
    }
  } else if (hasPatch || !isWholeDoc) {
    // Updating a map or table (with string key)
    if (firstOp || !patch.props.find(op.keyStr)) patch.props.set(op.keyStr, OMap<std::string, PVal>());
    if (hasPatch) patch.props[op.keyStr].set(patchKey, patchValue);
  }
}

struct AppliedChange { DecodedChange dc; std::vector<Op> ops; bool decoded = false; };

struct ChangeState {
  std::vector<AppliedChange*> changes; int64_t changeIndex = -1;
  size_t opIndex = 0; bool haveColumns = false; int64_t opCtr = 0;
  std::vector<int64_t> actorTable; int64_t actorIndex = -1;
  Op nextOp; bool hasNextOp = false; bool done = false;
  std::vector<std::string>* objectIds = nullptr;   // insertion-ordered Set
  void addObjectId(const std::string& id) { for (auto& s : *objectIds) if (s == id) return; objectIds->push_back(id); }
};

// new.js:1434-1451
static void getActorTable(DocState& ds, const DecodedChange& change, std::vector<int64_t>& actorTable) {
  if (ds.indexOfActor(change.actorIds[0]) < 0) {
    if (change.seq != 1) throw RangeError("Seq " + std::to_string(change.seq) + " is the first change for actor " + change.actorIds[0]);
    ds.actorIds.push_back(change.actorIds[0]);
  }
  actorTable.clear();
  for (auto& actorId : change.actorIds) {
    int64_t index = ds.indexOfActor(actorId);
    if (index < 0) throw RangeError("actorId " + actorId + " is not known to document");
    actorTable.push_back(index);
  }
}

// new.js:1387-1425 (column position checks are implied by the typed row layout)
static void updateBlockColumns(DocState& ds, const std::vector<Column>& changeCols) {
  for (auto& c : changeCols) {
    const int id = c.columnId;
    if (id == COL_PRED_NUM || id == COL_PRED_ACTOR || id == COL_PRED_CTR) continue;
    if (std::find(std::begin(DOC_OPS_COLUMN_IDS), std::end(DOC_OPS_COLUMN_IDS), id) != std::end(DOC_OPS_COLUMN_IDS)) continue;
    if (std::find(ds.extraColumnIds.begin(), ds.extraColumnIds.end(), id) == ds.extraColumnIds.end()) {
      ds.extraColumnIds.push_back(id); std::sort(ds.extraColumnIds.begin(), ds.extraColumnIds.end());
    }
  }
}

// new.js:678-724
static void readNextChangeOp(DocState& ds, ChangeState& cs) {
  while (cs.changeIndex < (int64_t)cs.changes.size() - 1 && (!cs.haveColumns || cs.opIndex >= cs.changes[cs.changeIndex]->ops.size())) {
    cs.changeIndex += 1;
    AppliedChange& change = *cs.changes[cs.changeIndex];
    updateBlockColumns(ds, change.dc.columns);
    getActorTable(ds, change.dc, cs.actorTable);
    if (!change.decoded) {
      change.ops = readAllOps(change.dc.columns, CHANGE_COLUMN_IDS, 16, 7, &cs.actorTable);
      change.decoded = true;
    }
    cs.haveColumns = true; cs.opIndex = 0; cs.opCtr = change.dc.startOp;
    if (change.ops.empty()) change.dc.maxOp = change.dc.startOp - 1;
    cs.actorIndex = ds.indexOfActor(change.dc.actorIds[0]);
  }
  if (cs.opIndex >= cs.changes[cs.changeIndex]->ops.size()) { cs.done = true; cs.hasNextOp = false; return; }
  cs.nextOp = cs.changes[cs.changeIndex]->ops[cs.opIndex++]; cs.hasNextOp = true;
  cs.nextOp.idActor = cs.actorIndex; cs.nextOp.idCtr = cs.opCtr;
  cs.changes[cs.changeIndex]->dc.maxOp = cs.opCtr;
  if (cs.opCtr > ds.maxOp) ds.maxOp = cs.opCtr;
  cs.opCtr += 1;
  const Op& op = cs.nextOp;
  auto s = [](int64_t v) { return v == NUL ? std::string("null") : std::to_string(v); };
  if ((op.objCtr == NUL && op.objActor != NUL) || (op.objCtr != NUL && op.objActor == NUL))
    throw RangeError("Mismatched object reference: (" + s(op.objCtr) + ", " + s(op.objActor) + ")");
  if ((op.keyCtr == NUL && op.keyActor != NUL) || (op.keyCtr == 0 && op.keyActor != NUL) || (op.keyCtr > 0 && op.keyActor == NUL))
    throw RangeError("Mismatched operation key: (" + s(op.keyCtr) + ", " + s(op.keyActor) + ")");
}

struct DocCursor { size_t blockIndex; size_t pos; };

// new.js:658-670
static bool readNextDocOp(const DocState& ds, DocCursor& cur, Op& out) {
  const Block* block = ds.blocks[cur.blockIndex].get();
  if (cur.pos < block->ops.size()) { out = block->ops[cur.pos++]; return true; }
  if (cur.blockIndex == ds.blocks.size() - 1) return false;
  cur.blockIndex += 1; cur.pos = 0; block = ds.blocks[cur.blockIndex].get();
  if (cur.pos < block->ops.size()) { out = block->ops[cur.pos++]; return true; }
  // the reference would read a row of nulls from an empty block; blocks after the first are never empty
  return false;
}

// new.js:1052-1290
static int64_t mergeDocChangeOps(Patches& patches, Block& newBlock, std::vector<Op>& outOps, ChangeState& cs, DocState& ds,
                                 int64_t listIndex, DocCursor& cur) {
  const Op firstOp = cs.nextOp; const bool insert = firstOp.insert;
  const int64_t objActor = firstOp.objActor, objCtr = firstOp.objCtr;
  const std::string objectId = objActor == NUL ? "_root" : opIdStr(objCtr, ds.actorOf(objActor));
  const int64_t idActorIndex = cs.actorIndex; const std::string idActor = ds.actorOf(idActorIndex);
  bool foundListElem = false, elemVisible = false; PropStates propState;
  Op docOp; bool hasDocOp = readNextDocOp(ds, cur, docOp);
  int64_t docOpsConsumed = hasDocOp ? 1 : 0;
  int64_t docOpOldSuccNum = hasDocOp ? docOp.succNum() : 0;
  std::vector<Op> changeOps; std::vector<std::vector<bool>> predSeen;
  bool hasLastChangeKey = false; std::string lastChangeKey;
  bool firstIteration = true; Op changeOp;
  cs.addObjectId(objectId);

  while (true) {
    if (changeOps.empty()) {
      foundListElem = false;
      while (!cs.done && cs.nextOp.idActor == idActorIndex && cs.nextOp.insert == insert &&
             cs.nextOp.objActor == firstOp.objActor && cs.nextOp.objCtr == firstOp.objCtr) {
        const Op& nextOp = cs.nextOp;
        const Op* lastOp = changeOps.empty() ? nullptr : &changeOps.back();
        bool isOverwrite = false;
        for (int64_t i = 0; i < nextOp.succNum(); i++)
          for (const Op& prevOp : changeOps)
            if (nextOp.succActor[i] == prevOp.idActor && nextOp.succCtr[i] == prevOp.idCtr) isOverwrite = true;

        if (firstIteration) {
          // First change operation in a mergeDocChangeOps call is always used
        } else if (insert && lastOp && !nextOp.hasKeyStr && nextOp.keyActor == lastOp->idActor && nextOp.keyCtr == lastOp->idCtr) {
          // Collect consecutive insertions
        } else if (!insert && lastOp && nextOp.hasKeyStr && lastOp->hasKeyStr && nextOp.keyStr == lastOp->keyStr && !isOverwrite) {
          // Collect several updates to the same key
        } else if (!insert && lastOp && !nextOp.hasKeyStr && !lastOp->hasKeyStr &&
                   nextOp.keyActor == lastOp->keyActor && nextOp.keyCtr == lastOp->keyCtr && !isOverwrite) {
          // Collect several updates to the same list element
        } else if (!insert && !lastOp && !nextOp.hasKeyStr && hasDocOp && docOp.insert && !docOp.hasKeyStr &&
                   docOp.idActor == nextOp.keyActor && docOp.idCtr == nextOp.keyCtr) {
          // updating several consecutive list elements
        } else if (!insert && !lastOp && nextOp.hasKeyStr && hasLastChangeKey && js_less(lastChangeKey, nextOp.keyStr)) {
          // several keys in ascending order
        } else break;
        firstIteration = false;

        hasLastChangeKey = nextOp.hasKeyStr; lastChangeKey = nextOp.keyStr;
        changeOps.push_back(cs.nextOp);
        predSeen.emplace_back((size_t)cs.nextOp.succNum(), false);
        readNextChangeOp(ds, cs);
      }
    }
    firstIteration = false;

    // NB `changeOp` persists from the previous iteration when changeOps is empty (new.js:1140)
    if (!changeOps.empty()) changeOp = changeOps[0];
    const bool inCorrectObject = hasDocOp && docOp.objActor == changeOp.objActor && docOp.objCtr == changeOp.objCtr;
    const bool keyMatches = hasDocOp && docOp.hasKeyStr && changeOp.hasKeyStr && docOp.keyStr == changeOp.keyStr;
    const bool listElemMatches = hasDocOp && !docOp.hasKeyStr && !changeOp.hasKeyStr &&
      ((!docOp.insert && docOp.keyActor == changeOp.keyActor && docOp.keyCtr == changeOp.keyCtr) ||
       (docOp.insert && docOp.idActor == changeOp.keyActor && docOp.idCtr == changeOp.keyCtr));

    if (changeOps.empty() && !(inCorrectObject && (keyMatches || listElemMatches))) break;

    bool takeDocOp = false; size_t takeChangeOps = 0;
    if (insert || !inCorrectObject || (!docOp.hasKeyStr && changeOp.hasKeyStr) ||
        (docOp.hasKeyStr && changeOp.hasKeyStr && js_less(changeOp.keyStr, docOp.keyStr))) {
      takeChangeOps = changeOps.size();
      if (!inCorrectObject && !foundListElem && !changeOp.hasKeyStr && !changeOp.insert)
        throw RangeError("could not find list element with ID: " + opIdStr(changeOp.keyCtr, ds.actorOf(changeOp.keyActor)));
    } else if (keyMatches || listElemMatches || foundListElem) {
      for (size_t opIndex = 0; opIndex < changeOps.size(); opIndex++) {
        const Op& op = changeOps[opIndex];
        for (int64_t i = 0; i < op.succNum(); i++) {
          if (op.succActor[i] == docOp.idActor && op.succCtr[i] == docOp.idCtr) {
            size_t j = 0;
            while (j < docOp.succCtr.size() && (docOp.succCtr[j] < op.idCtr ||
                   (docOp.succCtr[j] == op.idCtr && ds.actorOf(docOp.succActor[j]) < idActor))) j++;
            docOp.succCtr.insert(docOp.succCtr.begin() + j, op.idCtr);
            docOp.succActor.insert(docOp.succActor.begin() + j, idActorIndex);
            predSeen[opIndex][i] = true;
            break;
          }
        }
      }
      if (listElemMatches) foundListElem = true;

      if (foundListElem && !listElemMatches) {
        takeChangeOps = changeOps.size();
      } else if (changeOps.empty() || docOp.idCtr < changeOp.idCtr ||
                 (docOp.idCtr == changeOp.idCtr && ds.actorOf(docOp.idActor) < idActor)) {
        takeDocOp = true;
        updatePatchProperty(patches, &newBlock, objectId, docOp, ds, propState, listIndex, true, docOpOldSuccNum);
        for (int64_t i = (int64_t)changeOps.size() - 1; i >= 0; i--) {
          bool deleted = true;
          for (size_t j = 0; j < predSeen[i].size(); j++) if (!predSeen[i][j]) deleted = false;
          if (changeOps[i].action == A_DEL && deleted) { changeOps.erase(changeOps.begin() + i); predSeen.erase(predSeen.begin() + i); }
        }
      } else if (docOp.idCtr == changeOp.idCtr && ds.actorOf(docOp.idActor) == idActor) {
        throw RangeError("duplicate operation ID: " + opIdStr(changeOp.idCtr, idActor));
      } else {
        takeChangeOps = 1;
      }
    } else {
      takeDocOp = true;
    }

    // Not in the reference: with neither side taken nothing changes any more, i.e. the reference spins forever here. That
    // happens when an insertion's reference element has update rows on both sides of a block boundary: seekWithinBlock's
    // resumeInsertion path (new.js:59-73, 143-145) compares against object ids it never read and stops at the block start.
    if (!takeDocOp && takeChangeOps == 0) throw RangeError("oracle: the reference does not terminate on this input (mergeDocChangeOps makes no progress)");
    if (takeDocOp) {
      outOps.push_back(docOp);
      addBlockOperation(newBlock, docOp, ds, false);
      if (docOp.insert && elemVisible) { elemVisible = false; listIndex++; }
      if (docOp.succNum() == 0) elemVisible = true;
      newBlock.numOps++;
      hasDocOp = readNextDocOp(ds, cur, docOp);
      if (hasDocOp) { docOpsConsumed++; docOpOldSuccNum = docOp.succNum(); }
    }

    if (takeChangeOps > 0) {
      for (size_t i = 0; i < takeChangeOps; i++) {
        Op op = changeOps[i];
        for (size_t j = 0; j < predSeen[i].size(); j++)
          if (!predSeen[i][j]) throw RangeError("no matching operation for pred: " + opIdStr(op.succCtr[j], ds.actorOf(op.succActor[j])));
        // appendOperation: the change's pred columns are not document columns; a new row has succNum 0
        Op row = op; row.succActor.clear(); row.succCtr.clear();
        outOps.push_back(row);
        addBlockOperation(newBlock, row, ds, true);
        updatePatchProperty(patches, &newBlock, objectId, row, ds, propState, listIndex, false, 0);
        if (op.insert) { elemVisible = false; listIndex++; } else elemVisible = true;
      }
      changeOps.erase(changeOps.begin(), changeOps.begin() + takeChangeOps);
      predSeen.erase(predSeen.begin(), predSeen.begin() + takeChangeOps);
      newBlock.numOps += (int64_t)takeChangeOps;
    }
  }

  if (hasDocOp) { outOps.push_back(docOp); newBlock.numOps++; addBlockOperation(newBlock, docOp, ds, false); }
  return docOpsConsumed;
}

// new.js:1304-1380
static void applyOps(Patches& patches, ChangeState& cs, DocState& ds) {
  const Op& n = cs.nextOp; SeekOps ops;
  ops.objNull = n.objActor == NUL; ops.objActorNum = n.objActor; ops.objCtr = n.objCtr; if (!ops.objNull) ops.objActor = ds.actorOf(n.objActor);
  ops.keyActorNull = n.keyActor == NUL; ops.keyActorNum = n.keyActor; ops.keyCtr = n.keyCtr; if (!ops.keyActorNull) ops.keyActor = ds.actorOf(n.keyActor);
  ops.hasKeyStr = n.hasKeyStr; ops.keyStr = n.keyStr; ops.idActor = ds.actorOf(n.idActor); ops.idCtr = n.idCtr; ops.insert = n.insert;
  const int64_t keyActorNum = n.keyActor, keyCtr = n.keyCtr; const bool insert = n.insert;

  SeekPos sp = seekToOp(ds, ops);
  const size_t blockIndex = sp.blockIndex; const int64_t skipCount = sp.skipCount;
  const Block& block = *ds.blocks[blockIndex];
  const bool resetFirstVisible = (skipCount == 0) || (block.firstVisibleActor == UNDEF) ||
    (!insert && block.firstVisibleActor == keyActorNum && block.firstVisibleCtr == keyCtr);
  auto nbp = std::make_shared<Block>(); Block& newBlock = *nbp;
  memcpy(newBlock.bloom, block.bloom, sizeof(block.bloom));
  newBlock.numOps = skipCount; newBlock.hasLastKey = block.hasLastKey; newBlock.lastKey = block.lastKey;
  newBlock.numVisible = block.numVisible; newBlock.lastObjectActor = block.lastObjectActor; newBlock.lastObjectCtr = block.lastObjectCtr;
  newBlock.firstVisibleActor = resetFirstVisible ? UNDEF : block.firstVisibleActor;
  newBlock.firstVisibleCtr = resetFirstVisible ? UNDEF : block.firstVisibleCtr;

  // Copy the operations up to the insertion position
  std::vector<Op>& outOps = newBlock.ops;
  outOps.reserve(block.ops.size() + 8);
  outOps.assign(block.ops.begin(), block.ops.begin() + skipCount);

  DocCursor cur{blockIndex, (size_t)skipCount};
  const int64_t docOpsConsumed = mergeDocChangeOps(patches, newBlock, outOps, cs, ds, sp.visibleCount, cur);
  const size_t lastBlockIndex = cur.blockIndex;

  // Copy the remaining operations after the insertion position
  const Block& lastBlock = *ds.blocks[lastBlockIndex];
  int64_t copyAfterMerge = -skipCount - docOpsConsumed;
  for (size_t i = blockIndex; i <= lastBlockIndex; i++) copyAfterMerge += ds.blocks[i]->numOps;
  outOps.insert(outOps.end(), lastBlock.ops.begin() + cur.pos, lastBlock.ops.begin() + cur.pos + copyAfterMerge);
  newBlock.numOps += copyAfterMerge;
  if (cur.pos + copyAfterMerge != lastBlock.ops.size()) throw RangeError("excess ops in column");

  if (blockIndex == lastBlockIndex && newBlock.numOps <= MAX_BLOCK_SIZE) {
    if (copyAfterMerge > 0 && block.lastVisibleActor != UNDEF && block.lastVisibleCtr != UNDEF) {
      newBlock.lastVisibleActor = block.lastVisibleActor; newBlock.lastVisibleCtr = block.lastVisibleCtr;
    }
    ds.blocks[blockIndex] = nbp;
  } else {
    std::vector<BlockP> newBlocks = splitBlock(newBlock);
    ds.blocks.erase(ds.blocks.begin() + blockIndex, ds.blocks.begin() + lastBlockIndex + 1);
    ds.blocks.insert(ds.blocks.begin() + blockIndex, newBlocks.begin(), newBlocks.end());
  }
}

static void parseOpIdStr(const std::string& id, int64_t& ctr, std::string& actor) {
  size_t at = id.find('@');
  if (at == std::string::npos || at == 0) throw RangeError("Not a valid opId: " + id);
  for (size_t i = 0; i < at; i++) if (id[i] < '0' || id[i] > '9') throw RangeError("Not a valid opId: " + id);
  ctr = std::stoll(id.substr(0, at)); actor = id.substr(at + 1);
}

// new.js:1461-1528
static void setupPatches(Patches& patches, const std::vector<std::string>& objectIds, DocState& ds) {
  for (std::string objectId : objectIds) {
    auto mit = ds.objectMeta.find(objectId);
    if (mit == ds.objectMeta.end()) throw TypeError("unknown object " + objectId);
    const ObjMeta* meta = &mit->second; const ObjMeta* childMeta = nullptr; bool patchExists = false;
    while (true) {
      const OMap<std::string, ChildVal>* kids = childMeta ? meta->children.find(childMeta->parentKey) : nullptr;
      const bool hasChildren = childMeta && kids && kids->size() > 0;
      if (!patches.count(objectId)) patches[objectId] = emptyObjectPatch(objectId, meta->type, meta->typeNull);
      if (childMeta && hasChildren) {
        if (meta->type == "list" || meta->type == "text") {
          for (auto& edit : patches[objectId]->edits) if (edit.hasOpId && !edit.opId.empty() && kids->find(edit.opId)) patchExists = true;
          if (!patchExists) {
            SeekOps sk; std::string elemActor; int64_t elemCtr;
            parseOpIdStr(objectId, sk.objCtr, sk.objActor); parseOpIdStr(childMeta->parentKey, elemCtr, elemActor);
            sk.objNull = false; sk.keyActorNull = false; sk.keyActor = elemActor; sk.keyCtr = elemCtr;
            sk.objActorNum = ds.indexOfActor(sk.objActor); sk.keyActorNum = ds.indexOfActor(elemActor); sk.insert = false;
            SeekPos pos = seekToOp(ds, sk);
            for (auto& kv : kids->items) {
              PVal pv;
              if (kv.second.isObj) {
                if (!patches.count(kv.second.objectId)) patches[kv.second.objectId] = emptyObjectPatch(kv.second.objectId, kv.second.type, kv.second.typeNull);
                pv.obj = patches[kv.second.objectId];
              } else pv.prim = kv.second.prim;
              Edit e; e.action = Edit::UPDATE; e.index = pos.visibleCount; e.opId = kv.first; e.hasOpId = true; e.value = pv;
              appendEdit(patches[objectId]->edits, std::move(e));
            }
          }
        } else {
          OMap<std::string, PVal>& values = patches[objectId]->props[childMeta->parentKey];
          for (auto& kv : kids->items) {
            if (values.find(kv.first)) patchExists = true;
            else if (kv.second.isObj) {
              if (!patches.count(kv.second.objectId)) patches[kv.second.objectId] = emptyObjectPatch(kv.second.objectId, kv.second.type, kv.second.typeNull);
              PVal pv; pv.obj = patches[kv.second.objectId]; values.set(kv.first, pv);
            } else { PVal pv; pv.prim = kv.second.prim; values.set(kv.first, pv); }
          }
        }
      }
      if (patchExists || !meta->hasParent || (childMeta && !hasChildren)) break;
      childMeta = meta; objectId = meta->parentObj;
      auto pit = ds.objectMeta.find(objectId);
      if (pit == ds.objectMeta.end()) throw TypeError("unknown object " + objectId);
      meta = &pit->second;
    }
  }
}

// new.js:1604-1635
static PObjP documentPatch(DocState& ds) {
  PropStates propState; Patches patches;
  patches["_root"] = emptyObjectPatch("_root", "map", false);
  int64_t lastObjActor = NUL, lastObjCtr = NUL; std::string objectId = "_root"; bool elemVisible = false; int64_t listIndex = 0;
  for (auto& bp : ds.blocks) for (const Op& docOp : bp->ops) {
    if (docOp.objActor != lastObjActor || docOp.objCtr != lastObjCtr) {
      objectId = opIdStr(docOp.objCtr, ds.actorOf(docOp.objActor));
      lastObjActor = docOp.objActor; lastObjCtr = docOp.objCtr; propState.clear(); listIndex = 0; elemVisible = false;
    }
    if (docOp.insert && elemVisible) { elemVisible = false; listIndex++; }
    if (docOp.succNum() == 0) elemVisible = true;
    if (docOp.idCtr > ds.maxOp) ds.maxOp = docOp.idCtr;
    for (auto c : docOp.succCtr) if (c > ds.maxOp) ds.maxOp = c;
    updatePatchProperty(patches, nullptr, objectId, docOp, ds, propState, listIndex, true, docOp.succNum());
  }
  return patches["_root"];
}

struct PatchResult {
  int64_t maxOp = 0; std::map<std::string, int64_t> clock; std::vector<std::string> deps; int64_t pendingChanges = 0; PObjP diffs;
  bool hasActorSeq = false; std::string actor; int64_t seq = 0;
};

// class BackendDoc, new.js:1694-2069
struct BackendDoc {
  int64_t maxOp = 0; bool haveHashGraph = false;
  std::vector<std::string> changes;                       // binary changes in application order
  std::vector<bool> changePresent;
  std::unordered_map<std::string, int64_t> changeIndexByHash;
  std::unordered_map<std::string, std::vector<std::string>> dependenciesByHash, dependentsByHash;
  std::map<std::string, std::vector<std::string>> hashesByActor;
  std::vector<std::string> actorIds, heads; std::map<std::string, int64_t> clock;
  std::vector<std::shared_ptr<AppliedChange>> queue;
  std::map<std::string, ObjMeta> objectMeta;
  std::vector<BlockP> blocks; std::vector<int> extraColumnIds;
  std::string binaryDoc; bool hasBinaryDoc = false; PObjP initPatch;
  std::string extraBytes;
  // change metadata rows (the reference keeps these as encoders: changesEncoders)
  struct ChangeMeta { int64_t actor, seq, maxOp, time; std::string message; std::vector<int64_t> depsIndex; std::string extra; };
  std::vector<ChangeMeta> changeMetas;

  BackendDoc() {
    haveHashGraph = true;
    ObjMeta root; root.type = "map"; objectMeta["_root"] = root;
    blocks.push_back(std::make_shared<Block>());
  }

  // new.js:1709-1750 (load path) incl. readDocumentChanges new.js:1645-1675
  explicit BackendDoc(const std::string& buffer) {
    ObjMeta root; root.type = "map"; objectMeta["_root"] = root;
    DocHeader doc = decodeDocumentHeader(buffer);
    // readDocumentChanges
    { std::vector<Column> cols = doc.changesColumns;
      // decode change meta columns generically
      const std::string empty; auto bufOf = [&](int id) -> const std::string& { for (auto& c : cols) if (c.columnId == id) return c.buffer; return empty; };
      RLEDecoder actorD(T_UINT, bufOf(DCOL_ACTOR)); DeltaDecoder seqD(bufOf(DCOL_SEQ)), maxOpD(bufOf(DCOL_MAX_OP)), timeD(bufOf(DCOL_TIME));
      RLEDecoder msgD(T_UTF8, bufOf(DCOL_MESSAGE)), depsNumD(T_UINT, bufOf(DCOL_DEPS_NUM)); DeltaDecoder depsIndexD(bufOf(DCOL_DEPS_INDEX));
      RLEDecoder extraLenD(T_UINT, bufOf(DCOL_EXTRA_LEN)); Decoder extraRawD(bufOf(DCOL_EXTRA_RAW));
      std::vector<int64_t> actorNums; std::set<int64_t> headIndexes; int64_t numChanges = 0;
      while (!actorD.done()) {
        RV a = actorD.readValue(), s = seqD.readValue(), dn = depsNumD.readValue();
        ChangeMeta m; m.actor = a.null ? NUL : a.num; m.seq = s.null ? NUL : s.num;
        RV mo = maxOpD.readValue(), ti = timeD.readValue(), ms = msgD.readValue(), el = extraLenD.readValue();
        m.maxOp = mo.null ? NUL : mo.num; m.time = ti.null ? NUL : ti.num; m.message = ms.null ? "" : ms.str;
        if (!el.null) m.extra = extraRawD.readRawBytes((size_t)((uint64_t)el.num >> 4));
        if (m.actor < 0 || m.actor >= (int64_t)doc.actorIds.size()) throw RangeError("actor index out of range");
        const std::string& actorId = doc.actorIds[m.actor];
        int64_t expected = clock.count(actorId) ? clock[actorId] + 1 : -1;
        if (m.seq != 1 && m.seq != expected)
          throw RangeError("Expected seq " + (expected < 0 ? std::string("NaN") : std::to_string(expected)) + ", got " + std::to_string(m.seq) + " for actor " + actorId);
        actorNums.push_back(m.actor); clock[actorId] = m.seq; headIndexes.insert(numChanges);
        for (int64_t j = 0; j < (dn.null ? 0 : dn.num); j++) { RV di = depsIndexD.readValue(); m.depsIndex.push_back(di.null ? NUL : di.num); headIndexes.erase(di.num); }
        changeMetas.push_back(m); numChanges++;
      }
      std::vector<std::string> headActors; for (auto ix : headIndexes) headActors.push_back(doc.actorIds[actorNums[ix]]);
      std::sort(headActors.begin(), headActors.end());
      binaryDoc = buffer; hasBinaryDoc = true;
      changes.assign(numChanges, std::string()); changePresent.assign(numChanges, false);
      actorIds = doc.actorIds; heads = doc.heads; extraBytes = doc.extraBytes;
      if (doc.heads.size() == 1 && headActors.size() == 1) {
        auto& v = hashesByActor[headActors[0]]; v.assign(clock[headActors[0]], std::string()); v[clock[headActors[0]] - 1] = doc.heads[0];
      }
      if (doc.heads.size() == doc.headsIndexes.size()) { for (size_t i = 0; i < doc.heads.size(); i++) changeIndexByHash[doc.heads[i]] = doc.headsIndexes[i]; }
      else if (doc.heads.size() == 1) changeIndexByHash[doc.heads[0]] = numChanges - 1;
      else for (auto& h : doc.heads) changeIndexByHash[h] = -1;
    }
    auto blk = std::make_shared<Block>();
    blk->ops = readAllOps(doc.opsColumns, DOC_OPS_COLUMN_IDS, 16, 8, nullptr);
    for (auto& c : doc.opsColumns) if (std::find(std::begin(DOC_OPS_COLUMN_IDS), std::end(DOC_OPS_COLUMN_IDS), c.columnId) == std::end(DOC_OPS_COLUMN_IDS)) extraColumnIds.push_back(c.columnId);
    updateBlockMetadata(*blk);
    if (blk->numOps > MAX_BLOCK_SIZE) blocks = splitBlock(*blk); else blocks.push_back(blk);
    DocState ds; ds.blocks = blocks; ds.actorIds = actorIds; ds.objectMeta = objectMeta; ds.maxOp = 0;
    initPatch = documentPatch(ds); objectMeta = ds.objectMeta; maxOp = ds.maxOp;
  }

  // new.js:1550-1597
  void applyChangesPass(Patches& patches, std::vector<std::shared_ptr<AppliedChange>>& decodedChanges, DocState& ds,
                        std::vector<std::string>& objectIds, bool throwExceptions,
                        std::vector<std::shared_ptr<AppliedChange>>& applied, std::vector<std::shared_ptr<AppliedChange>>& enqueued) {
    std::set<std::string> headsSet(ds.heads.begin(), ds.heads.end()), batchHashes;
    std::map<std::string, int64_t> clk = ds.clock;
    for (auto& chp : decodedChanges) {
      const DecodedChange& change = chp->dc;
      if (ds.changeIndexByHash->count(change.hash) || batchHashes.count(change.hash)) continue;
      const int64_t expectedSeq = (clk.count(change.actor) ? clk[change.actor] : 0) + 1;
      bool causallyReady = true;
      for (auto& dep : change.deps) {
        auto it = ds.changeIndexByHash->find(dep);
        if ((it == ds.changeIndexByHash->end() || it->second == -1) && !batchHashes.count(dep)) causallyReady = false;
      }
      if (!causallyReady) enqueued.push_back(chp);
      else if (change.seq < expectedSeq) {
        if (throwExceptions) throw RangeError("Reuse of sequence number " + std::to_string(change.seq) + " for actor " + change.actor);
        applied.clear(); enqueued = decodedChanges; return;
      } else if (change.seq > expectedSeq) {
        throw RangeError("Skipped sequence number " + std::to_string(expectedSeq) + " for actor " + change.actor);
      } else {
        clk[change.actor] = change.seq; batchHashes.insert(change.hash);
        for (auto& dep : change.deps) headsSet.erase(dep);
        headsSet.insert(change.hash); applied.push_back(chp);
      }
    }
    if (!applied.empty()) {
      ChangeState cs; for (auto& a : applied) cs.changes.push_back(a.get()); cs.objectIds = &objectIds;
      readNextChangeOp(ds, cs);
      while (!cs.done) applyOps(patches, cs, ds);
      ds.heads.assign(headsSet.begin(), headsSet.end());   // std::set iterates sorted
      ds.clock = clk;
    }
  }

  // new.js:1797-1879
  PatchResult applyChanges(const std::vector<std::string>& changeBuffers, bool isLocal = false) {
    std::vector<std::shared_ptr<AppliedChange>> decodedChanges;
    for (auto& buf : changeBuffers) { auto a = std::make_shared<AppliedChange>(); a->dc = decodeChangeColumns(buf); decodedChanges.push_back(a); }
    Patches patches; patches["_root"] = emptyObjectPatch("_root", "map", false);
    std::unordered_map<std::string, int64_t> cibh = changeIndexByHash;
    DocState ds; ds.maxOp = maxOp; ds.changeIndexByHash = &cibh; ds.actorIds = actorIds; ds.heads = heads; ds.clock = clock;
    ds.blocks = blocks; ds.objectMeta = objectMeta; ds.extraColumnIds = extraColumnIds;
    std::vector<std::shared_ptr<AppliedChange>> q = decodedChanges; q.insert(q.end(), queue.begin(), queue.end());
    std::vector<std::shared_ptr<AppliedChange>> allApplied; std::vector<std::string> objectIds;
    while (true) {
      std::vector<std::shared_ptr<AppliedChange>> applied, enqueued;
      applyChangesPass(patches, q, ds, objectIds, haveHashGraph, applied, enqueued);
      q = enqueued;
      for (size_t i = 0; i < applied.size(); i++) cibh[applied[i]->dc.hash] = (int64_t)(changes.size() + allApplied.size() + i);
      allApplied.insert(allApplied.end(), applied.begin(), applied.end());
      if (q.empty()) break;
      if (applied.empty()) {
        if (haveHashGraph) break;
        computeHashGraph();   // new.js:1837-1839
        cibh = changeIndexByHash;
      }
    }
    setupPatches(patches, objectIds, ds);

    // Update the document state only if applyChanges did not throw
    for (auto& chp : allApplied) {
      const DecodedChange& change = chp->dc;
      changes.push_back(change.buffer); changePresent.push_back(true);
      auto& hv = hashesByActor[change.actor]; if ((int64_t)hv.size() < change.seq) hv.resize(change.seq); hv[change.seq - 1] = change.hash;
      changeIndexByHash[change.hash] = (int64_t)changes.size() - 1;
      dependenciesByHash[change.hash] = change.deps; dependentsByHash[change.hash];
      for (auto& dep : change.deps) dependentsByHash[dep].push_back(change.hash);
      // appendChange new.js:1680-1692
      ChangeMeta m; m.actor = ds.indexOfActor(change.actor);   // (actorIds holds each id once)
      m.seq = change.seq; m.maxOp = change.maxOp; m.time = change.time; m.message = change.message;
      for (auto& dep : change.deps) m.depsIndex.push_back(changeIndexByHash.count(dep) ? changeIndexByHash[dep] : NUL);
      m.extra = change.extraBytes; changeMetas.push_back(m);
    }
    maxOp = ds.maxOp; actorIds = ds.actorIds; heads = ds.heads; clock = ds.clock; blocks = ds.blocks; objectMeta = ds.objectMeta;
    extraColumnIds = ds.extraColumnIds; queue = q; hasBinaryDoc = false; binaryDoc.clear(); initPatch.reset();

    PatchResult r; r.maxOp = maxOp; r.clock = clock; r.deps = heads; r.pendingChanges = (int64_t)queue.size(); r.diffs = patches["_root"];
    if (isLocal && decodedChanges.size() == 1) { r.hasActorSeq = true; r.actor = decodedChanges[0]->dc.actor; r.seq = decodedChanges[0]->dc.seq; }
    return r;
  }

  // new.js:2060-2068
  PatchResult getPatch() {
    PatchResult r; r.maxOp = maxOp; r.clock = clock; r.deps = heads; r.pendingChanges = (int64_t)queue.size();
    if (initPatch) r.diffs = initPatch;
    else { DocState ds; ds.blocks = blocks; ds.actorIds = actorIds; ObjMeta root; root.type = "map"; ds.objectMeta["_root"] = root; ds.maxOp = 0; r.diffs = documentPatch(ds); }
    return r;
  }

  // new.js:2033-2055
  std::string save() {
    if (hasBinaryDoc) return binaryDoc;
    DocHeader doc;
    { RLEEncoder actorE(T_UINT), msgE(T_UTF8), depsNumE(T_UINT), extraLenE(T_UINT); DeltaEncoder seqE, maxOpE, timeE, depsIndexE; std::string extraRaw;
      for (auto& m : changeMetas) {
        actorE.appendValue(RV::Num(m.actor)); seqE.appendValue(RV::Num(m.seq)); maxOpE.appendValue(RV::Num(m.maxOp)); timeE.appendValue(RV::Num(m.time));
        msgE.appendValue(RV::Str(m.message)); depsNumE.appendValue(RV::Num((int64_t)m.depsIndex.size()));
        for (auto d : m.depsIndex) depsIndexE.appendValue(d == NUL ? RV() : RV::Num(d));
        extraLenE.appendValue(RV::Num(((int64_t)m.extra.size() << 4) | VT_BYTES)); extraRaw += m.extra;
      }
      doc.changesColumns = {{DCOL_ACTOR, actorE.finish()}, {DCOL_SEQ, seqE.finish()}, {DCOL_MAX_OP, maxOpE.finish()}, {DCOL_TIME, timeE.finish()},
                            {DCOL_MESSAGE, msgE.finish()}, {DCOL_DEPS_NUM, depsNumE.finish()}, {DCOL_DEPS_INDEX, depsIndexE.finish()},
                            {DCOL_EXTRA_LEN, extraLenE.finish()}, {DCOL_EXTRA_RAW, extraRaw}}; }
    std::vector<Op> all; for (auto& b : blocks) all.insert(all.end(), b->ops.begin(), b->ops.end());
    doc.opsColumns = encodeDocOps(all, extraColumnIds);
    doc.actorIds = actorIds; doc.heads = heads;
    for (auto& h : heads) doc.headsIndexes.push_back(changeIndexByHash.count(h) ? changeIndexByHash[h] : 0);
    doc.extraBytes = extraBytes;
    binaryDoc = encodeDocumentHeader(doc); hasBinaryDoc = true;
    return binaryDoc;
  }

  // new.js:1887-1912 computeHashGraph. The reference saves the document, decodes it again (decodeChanges -> decodeDocument,
  // columnar.js:1040-1047, 876-981) and re-encodes every change (encodeChange, columnar.js:710-738). What decodeDocument
  // would read back is exactly the change metadata and the document ops held here, so this starts from those.
  void computeHashGraph() {
    struct HOp {
      int64_t idCtr = 0, idActor = 0, objActor = NUL, objCtr = NUL, keyActor = NUL, keyCtr = NUL; bool hasKeyStr = false; std::string keyStr;
      bool insert = false; int64_t action = 0, valLen = 0; std::string valRaw; std::vector<std::pair<int64_t, int64_t>> pred; bool del = false;
    };
    const size_t numChanges = changeMetas.size();
    // ---- groupChangeOps (columnar.js:876-944)
    std::map<int64_t, std::vector<size_t>> changesByActor;
    for (size_t i = 0; i < numChanges; i++) {
      auto& list = changesByActor[changeMetas[i].actor];
      if (changeMetas[i].seq != (int64_t)list.size() + 1) throw RangeError("Expected seq = " + std::to_string(list.size() + 1) + ", got " + std::to_string(changeMetas[i].seq));
      if (changeMetas[i].seq > 1 && changeMetas[list.back()].maxOp > changeMetas[i].maxOp) throw RangeError("maxOp must increase monotonically per actor");
      list.push_back(i);
    }
    typedef std::pair<int64_t, int64_t> Id;   // (counter, actor index)
    std::map<Id, size_t> opsById; std::vector<HOp> ops;
    for (auto& b : blocks) for (auto& op : b->ops) {
      if (op.action == 3) throw RangeError("document should not contain del operations");
      HOp h; h.idCtr = op.idCtr; h.idActor = op.idActor; h.objActor = op.objActor; h.objCtr = op.objCtr; h.keyActor = op.keyActor; h.keyCtr = op.keyCtr;
      h.hasKeyStr = op.hasKeyStr; h.keyStr = op.keyStr; h.insert = op.insert; h.action = op.action; h.valLen = op.valLen == NUL ? 0 : op.valLen; h.valRaw = op.valRaw;
      const Id id(op.idCtr, op.idActor);
      auto it = opsById.find(id);
      if (it != opsById.end()) { h.pred = ops[it->second].pred; ops[it->second] = h; }   // a successor list mentioned it before it appeared
      else { opsById[id] = ops.size(); ops.push_back(h); }
      for (size_t k = 0; k < op.succCtr.size(); k++) {
        const Id sid(op.succCtr[k], op.succActor[k]);
        auto st = opsById.find(sid);
        if (st == opsById.end()) {
          HOp d; d.del = true; d.action = 3; d.idCtr = sid.first; d.idActor = sid.second; d.objActor = op.objActor; d.objCtr = op.objCtr;
          if (!op.hasKeyStr) { if (op.insert) { d.keyActor = op.idActor; d.keyCtr = op.idCtr; } else { d.keyActor = op.keyActor; d.keyCtr = op.keyCtr; } }
          else { d.hasKeyStr = true; d.keyStr = op.keyStr; }
          opsById[sid] = ops.size(); ops.push_back(d); st = opsById.find(sid);
        }
        ops[st->second].pred.push_back(id);
      }
    }
    std::vector<std::vector<size_t>> changeOps(numChanges);
    for (size_t o = 0; o < ops.size(); o++) {
      auto ca = changesByActor.find(ops[o].idActor);
      const std::string opIdText = std::to_string(ops[o].idCtr) + "@" + (ops[o].idActor >= 0 && (size_t)ops[o].idActor < actorIds.size() ? actorIds[ops[o].idActor] : std::string("?"));
      if (ca == changesByActor.end()) throw RangeError("Operation ID " + opIdText + " outside of allowed range");
      auto& list = ca->second; size_t left = 0, right = list.size();
      while (left < right) { const size_t mid = (left + right) / 2; if (changeMetas[list[mid]].maxOp < ops[o].idCtr) left = mid + 1; else right = mid; }
      if (left >= list.size()) throw RangeError("Operation ID " + opIdText + " outside of allowed range");
      changeOps[list[left]].push_back(o);
    }
    auto idLess = [&](const Id& a, const Id& b) { return a.first != b.first ? a.first < b.first : actorIds[a.second] < actorIds[b.second]; };
    // ---- decodeDocumentChanges (columnar.js:946-981) with encodeChange per change
    std::vector<std::string> newChanges(numChanges), newHashes(numChanges);
    std::set<std::string> headSet;
    for (size_t i = 0; i < numChanges; i++) {
      const ChangeMeta& m = changeMetas[i]; auto& mine = changeOps[i];
      std::sort(mine.begin(), mine.end(), [&](size_t a, size_t b) { return idLess(Id(ops[a].idCtr, ops[a].idActor), Id(ops[b].idCtr, ops[b].idActor)); });
      const int64_t startOp = m.maxOp - (int64_t)mine.size() + 1;
      for (size_t k = 0; k < mine.size(); k++) if (ops[mine[k]].idCtr != startOp + (int64_t)k || ops[mine[k]].idActor != m.actor)
        throw RangeError("Expected opId " + std::to_string(startOp + (int64_t)k) + "@" + actorIds[m.actor] + ", got " + std::to_string(ops[mine[k]].idCtr) + "@" + actorIds[ops[mine[k]].idActor]);
      std::vector<std::string> deps;
      for (int64_t index : m.depsIndex) {
        if (index < 0 || (size_t)index >= i || newHashes[index].empty()) throw RangeError("No hash for index " + std::to_string(index) + " while processing index " + std::to_string(i));
        deps.push_back(newHashes[index]); headSet.erase(newHashes[index]);
      }
      std::sort(deps.begin(), deps.end());
      // encodeChange (columnar.js:710-738) with parseAllOpIds (:132-170) and encodeOps (:370-436)
      std::set<std::string> actorSet;
      for (size_t o : mine) {
        const HOp& op = ops[o];
        if (op.objCtr != NUL) actorSet.insert(actorIds[op.objActor]);
        if (!op.hasKeyStr && op.keyActor != NUL) actorSet.insert(actorIds[op.keyActor]);
        for (auto& pr : op.pred) actorSet.insert(actorIds[pr.second]);
      }
      std::vector<std::string> localActors{actorIds[m.actor]};
      for (auto& a : actorSet) if (a != actorIds[m.actor]) localActors.push_back(a);
      auto localNum = [&](int64_t docActor) -> int64_t { for (size_t k = 0; k < localActors.size(); k++) if (localActors[k] == actorIds[docActor]) return (int64_t)k; throw RangeError("missing actorId"); };
      RLEEncoder objActorE(T_UINT), objCtrE(T_UINT), keyActorE(T_UINT), keyStrE(T_UTF8), actionE(T_UINT), valLenE(T_UINT), predNumE(T_UINT), predActorE(T_UINT);
      DeltaEncoder keyCtrE, predCtrE; BooleanEncoder insertE; std::string valRaw;
      for (size_t o : mine) {
        HOp& op = ops[o];
        if (op.objCtr == NUL) { objActorE.appendValue(RV()); objCtrE.appendValue(RV()); } else { objActorE.appendValue(RV::Num(localNum(op.objActor))); objCtrE.appendValue(RV::Num(op.objCtr)); }
        if (op.hasKeyStr) { keyActorE.appendValue(RV()); keyCtrE.appendValue(RV()); keyStrE.appendValue(RV::Str(op.keyStr)); }
        else if (op.keyActor == NUL) { keyActorE.appendValue(RV()); keyCtrE.appendValue(RV::Num(0)); keyStrE.appendValue(RV()); }   // _head
        else { keyActorE.appendValue(RV::Num(localNum(op.keyActor))); keyCtrE.appendValue(RV::Num(op.keyCtr)); keyStrE.appendValue(RV()); }
        insertE.appendValue(op.insert); actionE.appendValue(RV::Num(op.action));
        valLenE.appendValue(RV::Num(op.del ? 0 : op.valLen)); if (!op.del) valRaw += op.valRaw;   // (values travel as tag + bytes: canonical input re-encodes to itself)
        predNumE.appendValue(RV::Num((int64_t)op.pred.size()));
        std::sort(op.pred.begin(), op.pred.end(), idLess);
        for (auto& pr : op.pred) { predActorE.appendValue(RV::Num(localNum(pr.second))); predCtrE.appendValue(RV::Num(pr.first)); }
      }
      std::vector<Column> cols = {{COL_OBJ_ACTOR, objActorE.finish()}, {COL_OBJ_CTR, objCtrE.finish()}, {COL_KEY_ACTOR, keyActorE.finish()}, {COL_KEY_CTR, keyCtrE.finish()},
                                  {COL_KEY_STR, keyStrE.finish()}, {COL_INSERT, insertE.finish()}, {COL_ACTION, actionE.finish()}, {COL_VAL_LEN, valLenE.finish()},
                                  {COL_VAL_RAW, valRaw}, {0x70, predNumE.finish()}, {0x71, predActorE.finish()}, {0x73, predCtrE.finish()}};
      Encoder body; body.appendUint53((int64_t)deps.size()); for (auto& dep : deps) body.appendRaw(fromHex(dep));
      body.appendHexString(actorIds[m.actor]); body.appendUint53(m.seq); body.appendUint53(startOp); body.appendInt53(m.time); body.appendPrefixed(m.message);
      body.appendUint53((int64_t)localActors.size() - 1); for (size_t k = 1; k < localActors.size(); k++) body.appendHexString(localActors[k]);
      encodeColumnInfo(body, cols); for (auto& c : cols) body.appendRaw(c.buffer);
      body.appendRaw(m.extra);
      std::string hash; std::string bytes = encodeContainer(CHUNK_TYPE_CHANGE, body.buf, &hash);
      newHashes[i] = hash; newChanges[i] = bytes.size() >= DEFLATE_MIN_SIZE ? deflateChange(bytes) : bytes;
      headSet.insert(hash);
    }
    std::vector<std::string> actualHeads(headSet.begin(), headSet.end());
    if (actualHeads != heads) { std::string a, b; for (auto& h : heads) a += (a.empty() ? "" : ", ") + h; for (auto& h : actualHeads) b += (b.empty() ? "" : ", ") + h; throw RangeError("Mismatched heads hashes: expected " + a + ", got " + b); }
    // ---- new.js:1889-1911: the graph tables
    changes = newChanges; changePresent.assign(numChanges, true); changeIndexByHash.clear(); dependenciesByHash.clear(); dependentsByHash.clear(); hashesByActor.clear();
    std::map<std::string, int64_t> clk;
    for (size_t i = 0; i < numChanges; i++) {
      DecodedChange dc = decodeChangeColumns(changes[i]);
      changeIndexByHash[dc.hash] = (int64_t)i; dependenciesByHash[dc.hash] = dc.deps; dependentsByHash[dc.hash];
      for (auto& dep : dc.deps) dependentsByHash[dep].push_back(dc.hash);
      if (dc.seq == 1) hashesByActor[dc.actor].clear();
      hashesByActor[dc.actor].push_back(dc.hash);
      const int64_t expectedSeq = clk[dc.actor] + 1;
      if (dc.seq != expectedSeq) throw RangeError("Expected seq " + std::to_string(expectedSeq) + ", got seq " + std::to_string(dc.seq) + " from actor " + dc.actor);
      clk[dc.actor] = dc.seq;
    }
    haveHashGraph = true;
  }
  void requireHashGraph() { if (!haveHashGraph) computeHashGraph(); }

  // new.js:1921-1973
  std::vector<std::string> getChanges(const std::vector<std::string>& haveDeps) {
    requireHashGraph();
    if (haveDeps.empty()) return changes;
    std::vector<std::string> stack, toReturn; std::set<std::string> seen;
    for (auto& h : haveDeps) {
      seen.insert(h); auto it = dependentsByHash.find(h);
      if (it == dependentsByHash.end()) throw RangeError("hash not found: " + h);
      stack.insert(stack.end(), it->second.begin(), it->second.end());
    }
    while (!stack.empty()) {
      std::string hash = stack.back(); stack.pop_back(); seen.insert(hash); toReturn.push_back(hash);
      bool all = true; for (auto& dep : dependenciesByHash[hash]) if (!seen.count(dep)) all = false;
      if (!all) break;
      auto& ds_ = dependentsByHash[hash]; stack.insert(stack.end(), ds_.begin(), ds_.end());
    }
    bool headsSeen = true; for (auto& h : heads) if (!seen.count(h)) headsSeen = false;
    if (stack.empty() && headsSeen) { std::vector<std::string> out; for (auto& h : toReturn) out.push_back(changes[changeIndexByHash[h]]); return out; }
    stack = haveDeps; seen.clear();
    while (!stack.empty()) {
      std::string hash = stack.back(); stack.pop_back();
      if (!seen.count(hash)) {
        auto it = dependenciesByHash.find(hash); if (it == dependenciesByHash.end()) throw RangeError("hash not found: " + hash);
        stack.insert(stack.end(), it->second.begin(), it->second.end()); seen.insert(hash);
      }
    }
    std::vector<std::string> out;
    for (auto& c : changes) { DecodedChange dc = decodeChangeColumns(c); if (!seen.count(dc.hash)) out.push_back(c); }
    return out;
  }

  // new.js:1979-1997
  std::vector<std::string> getChangesAdded(BackendDoc& other) {
    requireHashGraph();
    std::vector<std::string> stack = heads, toReturn; std::set<std::string> seen;
    while (!stack.empty()) {
      std::string hash = stack.back(); stack.pop_back();
      if (!seen.count(hash) && !other.changeIndexByHash.count(hash)) {
        seen.insert(hash); toReturn.push_back(hash);
        auto& deps = dependenciesByHash[hash]; stack.insert(stack.end(), deps.begin(), deps.end());
      }
    }
    std::vector<std::string> out; for (auto it = toReturn.rbegin(); it != toReturn.rend(); ++it) out.push_back(changes[changeIndexByHash[*it]]);
    return out;
  }

  // new.js:2014-2028
  std::vector<std::string> getMissingDeps(const std::vector<std::string>& headsArg) {
    requireHashGraph();
    std::set<std::string> allDeps(headsArg.begin(), headsArg.end()), inQueue;
    for (auto& ch : queue) { inQueue.insert(ch->dc.hash); for (auto& dep : ch->dc.deps) allDeps.insert(dep); }
    std::vector<std::string> missing;
    for (auto& h : allDeps) if (!changeIndexByHash.count(h) && !inQueue.count(h)) missing.push_back(h);
    return missing;   // std::set iteration is already sorted
  }
};

}  // namespace orc
