"""Host-side mirror of ``rtabmap::VWDictionary`` and of the scoring half of ``rtabmap::Memory``
over the C ABI — same method names, argument meaning and error behaviour as the reference
(corelib/include/rtabmap/core/VWDictionary.h:46-160, corelib/src/VWDictionary.cpp), so the
parity tests read like tests of the reference class.  The C++ shim a maintainer would add to
RTAB-Map itself (``class VWDictionaryB200 : public VWDictionary``) is in INTEGRATION.md; this
file is the same thing for a Python host.  No computation happens here.
"""
from __future__ import annotations

import logging
from typing import Dict, List, Optional, Sequence

import numpy as np

from .capi import Engine, LcdError, LCD_DESC_F32, LCD_DESC_U8

log = logging.getLogger("rtabmap_b200")

# Parameters::k* keys and defaults used on this path (corelib/include/rtabmap/core/Parameters.h:243-264)
DEFAULT_PARAMETERS: Dict[str, str] = {
    "Kp/IncrementalDictionary": "true",
    "Kp/NndrRatio": "0.8",
    "Kp/NewWordsComparedTogether": "true",
    "Kp/NNStrategy": "0",  # exact linear search is the only strategy here (SURVEY.md F5)
    "Kp/TfIdfLikelihoodUsed": "true",
}


def _to_bool(v: str) -> bool:
    return str(v).lower() in ("1", "true", "yes")


class VWDictionaryB200:
    """Drop-in for VWDictionary: incremental / fixed visual vocabulary with exact k=2 NN + NNDR
    quantisation and the word -> signature inverted index, resident on one H100."""

    def __init__(self, parameters: Optional[Dict[str, str]] = None, device: int = 0, desc_type: int = LCD_DESC_U8,
                 desc_dim: int = 32, **engine_kwargs):
        self._engine = Engine(device=device, desc_type=desc_type, desc_dim=desc_dim, **engine_kwargs)
        self._incrementalDictionary = True
        self._nndrRatio = 0.8
        self._newWordsComparedTogether = True
        self.parseParameters(dict(DEFAULT_PARAMETERS, **(parameters or {})))

    # VWDictionary::parseParameters (VWDictionary.cpp:122-217)
    def parseParameters(self, parameters: Dict[str, str]):
        if "Kp/IncrementalDictionary" in parameters:
            self._incrementalDictionary = _to_bool(parameters["Kp/IncrementalDictionary"])
        if "Kp/NndrRatio" in parameters:
            self._nndrRatio = float(parameters["Kp/NndrRatio"])
        if "Kp/NewWordsComparedTogether" in parameters:
            self._newWordsComparedTogether = _to_bool(parameters["Kp/NewWordsComparedTogether"])
        if "Kp/NNStrategy" in parameters and int(parameters["Kp/NNStrategy"]) not in (0, 3, 4):
            log.warning("Kp/NNStrategy=%s is approximate in the reference; this engine is always exact (strategy 0 order)",
                        parameters["Kp/NNStrategy"])

    @property
    def engine(self) -> Engine:
        return self._engine

    def isIncremental(self) -> bool:
        return self._incrementalDictionary

    def setIncrementalDictionary(self):
        self._incrementalDictionary = True

    def setFixedDictionary(self, ids: Sequence[int], descriptors: np.ndarray):
        """VWDictionary::setFixedDictionary (VWDictionary.cpp:219-297) with the file already parsed:
        replaces the vocabulary by the given words and freezes it."""
        self.clear()
        self._engine.add_words(ids, descriptors)
        self._engine.last_word_id = int(max(ids)) if len(ids) else 0
        self._incrementalDictionary = False
        self.update()

    # VWDictionary::update (VWDictionary.cpp:475-701)
    def update(self):
        self._engine.update()

    # VWDictionary::addNewWords (VWDictionary.cpp:913-1229)
    def addNewWords(self, descriptors: np.ndarray, signatureId: int) -> List[int]:
        if descriptors is None or len(descriptors) == 0:
            log.error("Descriptors size is null!")
            return []
        if not self._incrementalDictionary and self._engine.size() == 0:
            log.error("Dictionary mode is set to fixed but no words are in it!")
            return []
        try:
            ids, _ = self._engine.quantize(descriptors, signatureId, self._incrementalDictionary, self._nndrRatio,
                                           self._newWordsComparedTogether)
        except LcdError as e:
            if e.code == -1:  # type / size mismatch: the reference logs and returns an empty list (:948-957)
                log.error(str(e))
                return []
            raise
        return [int(i) for i in ids]

    # VWDictionary::findNN (VWDictionary.cpp:1273-1552)
    def findNN(self, descriptors: np.ndarray) -> List[int]:
        if descriptors is None or len(descriptors) == 0:
            return []
        return [int(i) for i in self._engine.find_nn(descriptors, self._incrementalDictionary, self._nndrRatio)]

    # VWDictionary::addWord (VWDictionary.cpp:1554-1580)
    def addWord(self, wordId: int, descriptor: np.ndarray, references: Optional[Dict[int, int]] = None):
        self._engine.add_words([wordId], np.asarray(descriptor).reshape(1, -1))
        for sig, cnt in (references or {}).items():
            self._engine.add_refs(sig, [wordId] * cnt)

    # VWDictionary::addWordRef (VWDictionary.cpp:880-897)
    def addWordRef(self, wordId: int, signatureId: int) -> bool:
        if not self._engine.has_word(wordId):
            log.warning("Not found word %d (dict size=%d)", wordId, self._engine.size())
            return False
        self._engine.add_refs(signatureId, [wordId])
        return True

    def addSignatureRefs(self, signatureId: int, wordIds: Sequence[int]):
        """All addWordRef calls of one signature at once (Memory::enableWordsRef, Memory.cpp:6922-7035)."""
        self._engine.add_refs(signatureId, wordIds)

    # VWDictionary::removeAllWordRef for every word of a signature (Memory::disableWordsRef, Memory.cpp:6871-6897)
    def removeSignatureRefs(self, signatureId: int):
        self._engine.remove_sig(signatureId)

    # VWDictionary::removeWords (VWDictionary.cpp:1582-1593)
    def removeWords(self, wordIds: Sequence[int]):
        self._engine.remove_words(wordIds)

    def clear(self):
        self._engine.clear()

    def getLastWordId(self) -> int:
        return self._engine.last_word_id

    def getVisualWordsSize(self) -> int:
        return self._engine.size()

    def getIndexedWordsCount(self) -> int:
        return self._engine.indexed_size()

    def getNotIndexedWordsCount(self) -> int:
        return self._engine.not_indexed_size()

    def getTotalActiveReferences(self) -> int:
        return self._engine.total_refs()

    def getReferences(self, wordId: int) -> Dict[int, int]:
        s, c = self._engine.get_refs(wordId)
        return {int(a): int(b) for a, b in zip(s, c)}

    # Memory::computeLikelihood, TF-IDF branch (Memory.cpp:2215-2291)
    def computeLikelihood(self, signatureWordIds: Sequence[int], ids: Sequence[int], nSignatures: int) -> Dict[int, float]:
        if len(signatureWordIds) == 0:
            log.error("The signature is null")
            return {}
        if len(ids) == 0:
            log.warning("ids list is empty")
            return {}
        out = self._engine.score(signatureWordIds, ids, nSignatures)
        return {int(i): float(v) for i, v in zip(ids, out)}
