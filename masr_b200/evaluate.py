"""Batched evaluation over a manifest on the H100 path (SURVEY.md §8 f1): the decode + error-rate half of
``MASRTrainer.evaluate`` (masr/trainer.py:592-651; the loss half belongs to the training stack and is out of scope).

    error_rate, n = evaluate(predictor, read_manifest("dataset/manifest.test"), batch_size=32, metrics_type="cer")

``cer`` / ``wer`` restate masr/utils/metrics.py:4-29 (the reference calls the ``Levenshtein`` C extension; the edit distance
is computed here directly), ``labels_to_string`` restates masr/utils/utils.py:59-64.  Utterances go through
``MASRPredictor.predict_batches`` (pipelined staging); every utterance is decoded with B=1 semantics (DESIGN.md), whereas the
reference evaluates its zero-padded batch — the two agree on an un-padded batch.
"""
from __future__ import annotations

import json
from typing import Iterable, Iterator, List, Sequence, Tuple


def levenshtein(a: Sequence, b: Sequence) -> int:
    """Edit distance (insert / delete / substitute, unit costs) — what ``Levenshtein.distance`` returns."""
    if len(a) < len(b):
        a, b = b, a
    prev = list(range(len(b) + 1))
    for i, ca in enumerate(a, 1):
        cur = [i]
        for j, cb in enumerate(b, 1):
            cur.append(min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (ca != cb)))
        prev = cur
    return prev[-1]


def cer(prediction: str, label: str) -> float:
    """metrics.py:4-13: character error rate with blanks removed, normalised by the label length."""
    prediction, label = prediction.replace(" ", ""), label.replace(" ", "")
    return levenshtein(prediction, label) / float(len(label))


def wer(prediction: str, label: str) -> float:
    """metrics.py:16-29: words mapped to single symbols, then ``cer``."""
    pw, lw = prediction.split(" "), label.split(" ")
    ids = {}
    for s in pw + lw:
        ids.setdefault(s, len(ids))
    return levenshtein([ids[s] for s in pw], [ids[s] for s in lw]) / float(len(lw))


def labels_to_string(labels, vocabulary: Sequence[str], eos: int, blank_index: int = 0) -> List[str]:
    """utils.py:59-64: token id rows (padded with -1) -> text."""
    out = []
    for row in labels:
        out.append("".join(vocabulary[i] for i in row if i != blank_index and i != -1 and i != eos).replace("<space>", " "))
    return out


def read_manifest(path: str) -> Iterator[Tuple[str, str]]:
    """One JSON object per line with ``audio_filepath`` and ``text`` (data_utils/reader.py:55)."""
    with open(path, encoding="utf-8") as f:
        for line in f:
            line = line.strip()
            if line:
                d = json.loads(line)
                yield d["audio_filepath"], d["text"]


def evaluate(predictor, samples: Iterable[Tuple[object, str]], batch_size: int = 32, metrics_type: str = "cer",
             display_result: bool = False) -> Tuple[float, int]:
    """samples: (audio, reference text) pairs — audio is anything ``MASRPredictor.predict`` accepts.
    -> (mean error rate over the utterances as the reference averages it, trainer.py:649; number of utterances)."""
    if metrics_type not in ("cer", "wer"):
        raise ValueError("metrics_type must be 'cer' or 'wer'")
    metric = wer if metrics_type == "wer" else cer
    texts: List[List[str]] = []

    def batches():
        cur_a, cur_t = [], []
        for audio, text in samples:
            cur_a.append(audio)
            cur_t.append(text)
            if len(cur_a) == batch_size:
                texts.append(cur_t)
                yield cur_a
                cur_a, cur_t = [], []
        if cur_a:
            texts.append(cur_t)
            yield cur_a

    errors: List[float] = []
    for k, results in enumerate(predictor.predict_batches(batches())):
        for r, label in zip(results, texts[k]):
            e = metric(r["text"], label)
            errors.append(e)
            if display_result:
                print(f"预测结果为：{r['text']}\n实际标签为：{label}\n这条数据的{metrics_type}：{round(e, 6)}，"
                      f"当前{metrics_type}：{round(sum(errors) / len(errors), 6)}")
    return (float(sum(errors) / len(errors)) if errors else -1.0), len(errors)
