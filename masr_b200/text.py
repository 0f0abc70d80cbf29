"""Vocabulary handling (masr/data_utils/featurizer/text_featurizer.py:52-59): one ``token\\tcount``
per line, the line index is the token id; id 0 is ``<blank>``."""
from __future__ import annotations

from typing import List, Sequence


class TextFeaturizer:
    def __init__(self, vocab_filepath: str):
        self.unk = "<unk>"
        with open(vocab_filepath, "r", encoding="utf-8") as f:
            self._vocab_list = [line.split("\t")[0].replace("\n", "") for line in f.readlines()]
        self._vocab_dict = {tok: i for i, tok in enumerate(self._vocab_list)}

    @property
    def vocab_size(self) -> int:
        return len(self._vocab_list)

    @property
    def vocab_list(self) -> List[str]:
        return self._vocab_list

    def featurize(self, text: str) -> List[int]:
        out = []
        for tok in list(text.strip()):
            if tok == " ":
                tok = "<space>"
            out.append(self._vocab_dict.get(tok, self._vocab_dict.get(self.unk, 1)))
        return out


def ids_to_text(ids: Sequence[int], vocabulary: Sequence[str]) -> str:
    """ctc_greedy_decoder.py:26,31."""
    return "".join(vocabulary[i] for i in ids).replace("<space>", " ")


def nbest_dicts(hyps, vocabulary: Sequence[str]) -> List[dict]:
    """[(token ids, score)], best first -> the ``'n_best'`` entries [{'text', 'score'}] of a result."""
    return [{"text": ids_to_text(t, vocabulary), "score": float(s)} for t, s in hyps]
