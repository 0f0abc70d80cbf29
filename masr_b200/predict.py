"""Drop-in for ``masr.predict.MASRPredictor`` (masr/predict.py:19-362) on the H100 engine.

Same constructor arguments, same ``predict`` / ``predict_stream`` / ``reset_stream`` signatures,
same ``{'text': str, 'score': float}`` results, same YAML keys (``use_model``, ``streaming``,
``decoder``, ``preprocess_conf``, ``dataset_conf.dataset_vocab``) and the same ``inference.pt``
weights.  What changes is where the work happens: the waveform goes to the GPU once and only token
ids + a score come back (the reference featurises on the CPU, copies features up, copies the whole
[T,V] posterior down and decodes with numpy — predict.py:181-190, inference_predictor.py:59-64).

Additive entry points (the reference API is single-utterance): ``predict_batch``.
Hotwords (``decoder: ctc_beam_search`` only): ``MASRPredictor(..., hotwords=[...], hotword_score=1.5)`` boosts those words
inside the GPU prefix beam search (masr_b200/hotwords.py) for every call; ``predict``, ``predict_batch`` and
``predict_long`` take a per-call ``hotwords=`` that overrides the list (``[]``: none), and each slot of
``create_stream_pool`` can have its own (``StreamPool.set_hotwords``).  Scores never include the hotword credit.
N-best (``decoder: ctc_beam_search`` only): ``predict``, ``predict_batch`` and ``predict_stream`` take ``n_best=``, and
``create_stream_pool`` takes it for every slot; the result then also carries ``'n_best'``, the best hypotheses of the
search as ``[{'text', 'score'}, ...]``, best first, entry 0 the result's own text and score.
Audio at other sample rates than 16 kHz is resampled on the GPU, as the reference's featurizer does
(audio_featurizer.py:45-47), when the predictor is built with ``resample=True``; by default a rate mismatch raises.
Out of the hot-path scope and therefore explicit errors here: punctuation (``use_pun``), inverse
text normalisation (``is_itn``), model download (``configs=None``) and ``use_gpu=False`` (there is no CPU path).
"""
from __future__ import annotations

import logging
import os
from typing import List, Optional, Sequence

import numpy as np
import torch
import yaml

from . import SUPPORT_MODEL
from .audio import load_audio, pcm_bytes_to_float32, samples_to_float32
from .engine import ConformerEngine, EfficientConformerEngine, greedy_score, subsampled_len
from .resample import MODEL_RATE, needs_resampling
from .beam import check_n_best
from .text import TextFeaturizer, ids_to_text, nbest_dicts
from . import timestamps as ts

logger = logging.getLogger(__name__)


class _Cfg(dict):
    """``dict_to_object`` (masr/utils/utils.py:45-56): attribute access over nested dicts."""
    __setattr__ = dict.__setitem__
    __getattr__ = dict.__getitem__


def dict_to_object(obj):
    if not isinstance(obj, dict):
        return obj
    out = _Cfg()
    for k, v in obj.items():
        out[k] = dict_to_object(v)
    return out


# streaming window arithmetic of predict.py:283-289
DECODING_CHUNK_SIZE = 16
CONTEXT = 7
SUBSAMPLING = 4
CACHED_FEATURE_NUM = CONTEXT - SUBSAMPLING                         # 3 feature frames carried over
DECODING_WINDOW = (DECODING_CHUNK_SIZE - 1) * SUBSAMPLING + CONTEXT  # 67
STRIDE = SUBSAMPLING * DECODING_CHUNK_SIZE                         # 64


def chunk_starts(num_frames: int, is_end: bool) -> List[int]:
    """Start indices of the encoder chunks the reference runs for ``num_frames`` cached feature
    frames (predict.py:292-303); empty when it would return ``None``."""
    if num_frames < DECODING_WINDOW and not is_end:
        return []
    if num_frames < CONTEXT:
        return []
    left = CONTEXT if is_end else DECODING_WINDOW
    return list(range(0, num_frames - left + 1, STRIDE))


class MASRPredictor:
    _hotwords = None                      # the predictor's HotwordGraph (None: no hotwords)

    def __init__(self,
                 configs=None,
                 model_tag='conformer_streaming_fbank_aishell',
                 model_path='models/conformer_streaming_fbank/inference.pt',
                 use_pun=False,
                 pun_model_dir='models/pun_models/',
                 use_gpu=True,
                 resample=False,
                 hotwords=None,
                 hotword_score=1.5):
        """``resample``: accept audio at any sample rate and resample it to ``preprocess_conf.sample_rate`` on the GPU,
        as the reference's featurizer does (audio_featurizer.py:45-47); False keeps a rate mismatch an error.
        ``hotwords``: strings the prefix beam search boosts by ``hotword_score`` per token of every whole hotword a
        hypothesis contains (longest match; nested hotwords both count); None or ``[]``: no hotwords, the search as
        without.  A ValueError for hotwords with ``decoder: ctc_greedy``, for a character outside the vocabulary, and for
        an empty or over-32-token hotword.  The default score of 1.5 is untuned: pick it on your own data."""
        if not configs:
            raise Exception("masr_b200: model download (configs=None, model_tag=...) is not supported; "
                            "pass a YAML path or dict plus model_path")
        if isinstance(configs, str):
            with open(configs, 'r', encoding='utf-8') as f:
                configs = yaml.load(f.read(), Loader=yaml.FullLoader)
        self.configs = dict_to_object(configs)
        assert self.configs.use_model in SUPPORT_MODEL, f'没有该模型：{self.configs.use_model}'
        if not use_gpu:
            raise Exception("masr_b200 has no CPU path: use_gpu=False is not supported")
        if use_pun:
            raise Exception("masr_b200: the punctuation model (use_pun) is outside the hot-path scope")
        self.running = False
        self.use_gpu = use_gpu
        self._text_featurizer = TextFeaturizer(vocab_filepath=self.configs.dataset_conf.dataset_vocab)
        pc = self.configs.preprocess_conf
        if pc.get('feature_method', 'fbank') != 'fbank' or int(pc.get('n_mels', 80)) != 80:
            raise Exception("masr_b200 implements the fbank/80-mel front-end of the shipped configs only")
        self._sample_rate = int(pc.get('sample_rate', 16000))
        self._use_db = bool(pc.get('use_dB_normalization', True))
        self._target_db = float(pc.get('target_dB', -20))
        self._resample = bool(resample)
        if self._resample and self._sample_rate != MODEL_RATE:
            raise Exception(f"masr_b200 resamples to {MODEL_RATE} Hz only (preprocess_conf.sample_rate = {self._sample_rate})")
        self._beam_conf = None
        self.lm = None
        if self.configs.decoder == 'ctc_beam_search':
            # GPU prefix beam search: whole-utterance calls (engine.ctc_beam) and streaming (engine.StreamBeam =
            # BeamSearchDecoder.decode_chunk / reset_decoder).  With an ARPA file at language_model_path the LM (character-based,
            # or word-based with its lexicon when the vocabulary has <space>) is fused into the search (the reference's
            # Scorer, beam_search_decoder.py:28-37) and the score is approx_ctc; otherwise the search runs without LM and
            # reports the beam's log score.
            bc = dict(self.configs.get('ctc_beam_search_decoder_conf', {}) or {})
            self._beam_conf = {'beam_size': int(bc.get('beam_size', 300)), 'cutoff_prob': float(bc.get('cutoff_prob', 0.99)),
                               'cutoff_top_n': int(bc.get('cutoff_top_n', 40))}
            self.lm = self._load_lm(bc)
            if self.lm is not None:
                self._beam_conf.update(lm=self.lm, alpha=float(bc.get('alpha', 0.0)), beta=float(bc.get('beta', 0.0)))
        self._hotword_score = float(hotword_score)
        self._hotword_graphs = {}
        self._hotwords = self._graph(hotwords)
        if not os.path.exists(model_path):
            raise Exception("模型文件不存在，请检查{}是否存在！".format(model_path))
        from .squeezeformer import SqueezeformerEngine
        from .deepspeech2 import DeepSpeech2Engine
        engines = {'conformer': ConformerEngine, 'efficient_conformer': EfficientConformerEngine,
                   'squeezeformer': SqueezeformerEngine, 'deepspeech2': DeepSpeech2Engine}
        if self.configs.use_model not in engines:
            raise Exception(f"masr_b200: model '{self.configs.use_model}' is not implemented yet "
                            f"(available: {sorted(engines)})")
        self.predictor = engines[self.configs.use_model](model_path, streaming=bool(self.configs.streaming))
        self._can_stream = self.configs.use_model in ('conformer', 'deepspeech2', 'squeezeformer', 'efficient_conformer')
        if self.predictor.V != self._text_featurizer.vocab_size:
            raise Exception(f"vocabulary has {self._text_featurizer.vocab_size} entries but the model's CTC head has "
                            f"{self.predictor.V}")
        # streaming state (predict.py:70-73)
        self.remained_wav: Optional[np.ndarray] = None
        self.cached_feat: Optional[torch.Tensor] = None       # device [n, 80]
        self._stream = self.predictor.new_stream() if (self.configs.streaming and self._can_stream) else None
        self._hist_ids: List[int] = []
        self._hist_probs: List[np.float32] = []
        self._sbeam = None                                   # streaming beam-search state (created on the first chunk)
        self._sbeam_result = ([], 0.0)
        # warm-up, as the reference does (predict.py:88-93)
        warmup_audio = np.random.uniform(low=-2.0, high=2.0, size=(134240,))
        self.predict(audio_data=warmup_audio, is_itn=False)
        self.reset_stream()

    # ---------------------------------------------------------------------------------------------
    def _load_lm(self, bc):
        """The LM at ``language_model_path`` when that is a plain-text ARPA file (judged by content, not by extension),
        loaded once: a CharLM for a character-based file, a WordLM (lexicon-constrained, scored per word) for a word-based
        one when the vocabulary has ``<space>``; else None with a warning that names the reason."""
        from .lm import CharLM, WordLM, sniff
        path = bc.get('language_model_path') or ''
        kind = sniff(path)
        reason = {'missing': f'language model {path!r} not found',
                  'kenlm_binary': f'{path!r} is a KenLM binary; only plain-text ARPA language models are read',
                  'unknown': f'{path!r} is not an ARPA file'}.get(kind)
        lm = None
        if reason is None:
            vocab = self._text_featurizer.vocab_list
            lm = CharLM(path, vocab)
            if not lm.is_character_based:
                if '<space>' not in vocab:
                    reason, lm = f'{path!r} is a word-based LM and the vocabulary has no <space> token', None
                else:
                    lm = WordLM(path, vocab)
        if lm is None:
            logger.warning(f'ctc_beam_search: {reason}: GPU prefix beam search without LM (alpha/beta ignored)')
            return None
        logger.info(f'language model: model path = {path}, {lm.describe()}')
        return lm

    def _graph(self, hotwords):
        """A list of hotwords -> its HotwordGraph (built and checked once per distinct list), None for None or ``[]``."""
        from .hotwords import HotwordGraph, check_score, outside_lexicon
        if hotwords is None or len(hotwords) == 0:
            return None
        if self._beam_conf is None:
            raise ValueError("hotwords need the prefix beam search (decoder: ctc_beam_search), not ctc_greedy")
        check_score(self._hotword_score)
        key = tuple(hotwords)
        g = self._hotword_graphs.get(key)
        if g is None:
            vocab = self._text_featurizer.vocab_list
            g = HotwordGraph(hotwords, vocab, self._hotword_score)
            if getattr(self.lm, "BEAM", "") == "masr_ctc_prefix_beam_wordlm":
                missing = outside_lexicon(g, vocab, self.lm)
                if missing:
                    logger.warning(f"hotwords: the word LM's lexicon lacks {missing}: hotwords using them are never produced")
            if len(self._hotword_graphs) >= 16:
                self._hotword_graphs.pop(next(iter(self._hotword_graphs)))
            self._hotword_graphs[key] = g
        return g

    def _call_graph(self, hotwords):
        """The per-call ``hotwords=``: None keeps the predictor's list, a list (``[]`` included) replaces it."""
        return self._hotwords if hotwords is None else self._graph(hotwords)

    def _n_best(self, n_best):
        """The per-call ``n_best``: None, or an int in 1..beam_size (a ValueError otherwise, and for greedy decoding)."""
        if n_best is None:
            return None
        if self._beam_conf is None:
            raise ValueError("n_best needs the prefix beam search (decoder: ctc_beam_search), not ctc_greedy")
        return check_n_best(n_best, self._beam_conf['beam_size'])

    def _check_rate(self, sr):
        if sr != self._sample_rate and not self._resample:
            raise Exception(f"masr_b200: resampling is outside the hot-path scope (got {sr} Hz, model expects "
                            f"{self._sample_rate} Hz)")

    def _load_batch(self, audio_list, sample_rate):
        """-> (float32 waveforms, their rates or None when every row is at the model rate)."""
        waves, rates = [], []
        for a in audio_list:
            s, sr = load_audio(a, sample_rate)
            self._check_rate(sr)
            waves.append(s)
            rates.append(sr)
        return waves, (rates if needs_resampling(rates) else None)

    def _finish(self, text, use_pun, is_itn):
        if use_pun:
            logger.warning('标点符号模型没有初始化！')
        if is_itn:
            raise Exception("masr_b200: inverse text normalisation (is_itn) is outside the hot-path scope")
        return text

    def predict(self, audio_data, use_pun=False, is_itn=False, sample_rate=16000, timestamps=False, hotwords=None,
                n_best=None):
        """Whole-utterance recognition (predict.py:167-192).  ``timestamps``: the result also carries ``'tokens'``
        (``[{'token', 'start', 'end'}]``, seconds) and, when the vocabulary has ``<space>``, ``'words'``
        (masr_b200/timestamps.py).  ``hotwords``: this call's list (None: the predictor's; ``[]``: none).
        ``n_best`` (1..beam_size): the result also carries ``'n_best'``, at most ``n_best`` hypotheses ``{'text',
        'score'}`` in the order the search ranks them, entry 0 the result itself.  Their scores are what ``'score'`` is:
        the log probability, or approx_ctc with an LM (the ranking is by the fused score then, so those need not
        decrease down the list).  Timestamps are only for the result itself."""
        n_best = self._n_best(n_best)
        r = self._recognise(*self._load_batch([audio_data], sample_rate), timestamps, hotwords=self._call_graph(hotwords),
                            n_best=n_best)[0]
        r['text'] = self._finish(r['text'], use_pun, is_itn)
        return r

    def predict_batch(self, audio_list: Sequence, sample_rate=16000, timestamps=False, hotwords=None, n_best=None):
        """Additive: a list of utterances in one GPU pass; element i equals ``predict(audio_list[i])``.  With
        ``resample=True`` the rows may have different rates (WAV files carry their own).  ``timestamps``, ``hotwords``,
        ``n_best``: as in predict."""
        n_best = self._n_best(n_best)
        return self._recognise(*self._load_batch(audio_list, sample_rate), timestamps, hotwords=self._call_graph(hotwords),
                               n_best=n_best)

    def _recognise(self, waves, rates, timestamps=False, offsets=None, hotwords=None, n_best=None):
        """Waveforms -> ``[{'text', 'score'}]`` (+ token and word times, shifted by ``offsets[i]`` seconds; + ``'n_best'``)."""
        vocab = self._text_featurizer.vocab_list
        dt = ts.frame_seconds(self.predictor)
        offsets = offsets or [0.0] * len(waves)
        if self._beam_conf is not None:
            out = self.predictor.transcribe_beam(waves, use_db_normalization=self._use_db, target_db=self._target_db,
                                                 rates=rates, onsets=timestamps, hotwords=hotwords, n_best=n_best,
                                                 **self._beam_conf)
            res = [{'text': ids_to_text(t, vocab), 'score': s} for t, s in zip(out[0], out[1])]
            if timestamps:
                for r, t, f, off in zip(res, out[0], out[2], offsets):
                    ts.beam_result(r, t, f, vocab, dt, off)
            if n_best is not None:
                for r, hyps in zip(res, out[-1]):
                    r['n_best'] = nbest_dicts(hyps, vocab)
            return res
        g = self.predictor.transcribe(waves, self._use_db, self._target_db, return_frames=timestamps, rates=rates)
        self._raise_status(g.status)
        res = [{'text': ids_to_text(t, vocab), 'score': s} for t, s in zip(g.tokens, g.scores)]
        if timestamps:
            for b, (r, off) in enumerate(zip(res, offsets)):
                ids = g.frame_ids[b, :g.frame_lens[b]] if g.frame_ids is not None else []
                ts.greedy_result(r, ids, vocab, dt, off)
        return res

    def predict_batches(self, batches, sample_rate=16000, device_hook=None):
        """Additive: a stream of batches (iterable of lists of utterances) -> one list of ``{'text','score'}`` per batch, in
        order; element i of batch k equals ``predict(batches[k][i])``.  Host staging and the H2D copy of batch k+1 overlap
        the GPU pass of batch k (``ConformerEngine.transcribe_pipelined``), so the results lag the input by one batch.
        Greedy decoding only.  ``device_hook``: see ``transcribe_pipelined`` (cross-rank gather of a sharded deployment)."""
        vocab = self._text_featurizer.vocab_list
        if self._beam_conf is not None:
            # the prefix beam search of batch k runs on a second stream under the encoder of batch k+1
            loaded_b = (self._load_batch(audio_list, sample_rate) for audio_list in batches)
            for toks, scores in self.predictor.transcribe_beam_pipelined(loaded_b, use_db_normalization=self._use_db,
                                                                         target_db=self._target_db, with_rates=True,
                                                                         hotwords=self._hotwords, **self._beam_conf):
                yield [{'text': ids_to_text(t, vocab), 'score': s} for t, s in zip(toks, scores)]
            return

        loaded = (self._load_batch(audio_list, sample_rate) for audio_list in batches)
        for res in self.predictor.transcribe_pipelined(loaded, self._use_db, self._target_db, device_hook=device_hook,
                                                       with_rates=True):
            self._raise_status(res.status)
            yield [{'text': ids_to_text(t, vocab), 'score': s} for t, s in zip(res.tokens, res.scores)]

    @staticmethod
    def _raise_status(status):
        if status is not None and np.any(status != 0):
            # AudioSegment.normalize raises ValueError when gain > max_gain_db (audio.py:301-303)
            raise ValueError("无法将段规范化到目标dB，音频增益已经超过max_gain_db (300.0dB)")

    def init_vad(self, vad_predictor=None, vad_model_path=None):
        """predict.py:139-142.  ``vad_predictor``: any object with the reference's ``get_speech_timestamps(samples,
        sampling_rate)``; else the silero ONNX model at ``vad_model_path``, run on the GPU (masr_b200.vad.GpuSileroVAD)."""
        if vad_predictor is not None:
            self.vad_predictor = vad_predictor
        elif getattr(self, "vad_predictor", None) is None:
            if vad_model_path is None:
                raise Exception("masr_b200: predict_long needs a VAD: pass vad_predictor=... (an object with "
                                "get_speech_timestamps) or vad_model_path=<silero_vad.onnx>")
            from .vad import GpuSileroVAD
            self.vad_predictor = GpuSileroVAD(vad_model_path, device=self.predictor.device)

    def predict_long(self, audio_data, use_pun=False, is_itn=False, sample_rate=16000, vad_predictor=None, vad_model_path=None,
                     timestamps=False, hotwords=None):
        """Long-form recognition (predict.py:195-234): VAD segments -> recognise -> join with '，' and average the scores.
        All segments of the recording go through ONE batched GPU pass (``predict_batch``) instead of the reference's
        one-``predict``-per-segment loop; each segment's result equals ``predict(segment)`` (B=1 semantics).
        ``timestamps``: the result also carries ``'sentences'``, one ``{'text', 'score', 'start', 'end', 'tokens'}`` (+
        ``'words'``) per segment with non-empty text: the segment's bounds and its token times, in seconds of the
        recording.  ``hotwords``: as in predict, for every segment."""
        graph = self._call_graph(hotwords)
        self.init_vad(vad_predictor, vad_model_path)
        samples, sr = load_audio(audio_data, sample_rate)
        self._check_rate(sr)
        if sr != self._sample_rate:
            # predict.py:212-213: the whole recording is resampled first (on the GPU); the VAD runs on the 16 kHz samples
            samples, sr = self.predictor.resample([samples], [sr])[0], self._sample_rate
        stamps = self.vad_predictor.get_speech_timestamps(samples, sr)
        segs = [samples[t['start']:t['end']] for t in stamps]
        offsets = [t['start'] / sr for t in stamps]
        results = self._recognise(*self._load_batch(segs, sr), timestamps, offsets, graph) if segs else []
        texts, scores = '', []
        for r in results:
            if r['text'] != '':
                texts = texts + r['text'] if use_pun else texts + '，' + r['text']
            scores.append(r['score'])
        if texts[:1] == '，':
            texts = texts[1:]
        if use_pun and len(texts) > 0:
            logger.warning('标点符号模型没有初始化！')
        if is_itn:
            raise Exception("masr_b200: inverse text normalisation (is_itn) is outside the hot-path scope")
        out = {'text': texts, 'score': round(sum(scores) / len(scores), 2) if scores else 0}
        if timestamps:
            out['sentences'] = ts.sentences([(t['start'], t['end']) for t in stamps], results, sr)
        return out

    # ---------------------------------------------------------------------------------------------
    def predict_stream(self, audio_data, is_end=False, use_pun=False, is_itn=False, channels=1, samp_width=2,
                       sample_rate=16000, timestamps=False, n_best=None):
        """Streaming recognition, one push of audio per call (predict.py:237-343).  Returns ``None``
        while fewer than 67 feature frames are buffered, else the running ``{'text','score'}``; ``timestamps``: with
        ``'tokens'`` (+ ``'words'``) as in predict, timed since the last ``reset_stream``; ``n_best``: with ``'n_best'`` as
        in predict, over the frames seen so far."""
        if not self.configs.streaming:
            raise Exception(
                f"不支持改该模型流式识别，当前模型：{self.configs.use_model}，参数streaming为：{self.configs.streaming}")
        if not self._can_stream:
            raise NotImplementedError(f"masr_b200: predict_stream is not implemented for '{self.configs.use_model}' yet")
        if isinstance(audio_data, np.ndarray):
            new = samples_to_float32(audio_data)
        elif isinstance(audio_data, bytes):
            new = pcm_bytes_to_float32(audio_data, channels=channels, samp_width=samp_width)
        else:
            raise Exception(f'不支持该数据类型，当前数据类型为：{type(audio_data)}')
        self._check_rate(sample_rate)
        n_best = self._n_best(n_best)
        self.remained_wav = new if self.remained_wav is None else np.concatenate([self.remained_wav, new])
        if sample_rate != self._sample_rate:
            # predict.py:267-274: the buffer (the carried-over tail, already at 16 kHz, plus the new chunk) is labelled with
            # the chunk's rate and resampled as a whole on every push, as the reference does
            self.remained_wav = self.predictor.resample([self.remained_wav], [sample_rate])[0]

        # featurise everything not yet consumed; the reference dB-normalises the remainder IN PLACE on
        # every push (predict.py:274 + audio_featurizer.py:49-50), so the carried-over tail keeps the gain
        eng = self.predictor
        feats, frames, status = eng.fbank([self.remained_wav], self._use_db, self._target_db)
        gain = float(eng.last_gain.cpu().numpy()[0]) if self._use_db else 1.0
        self._raise_status(status.cpu().numpy())
        nf = frames[0]
        x_chunk = feats[0, :nf]
        self.cached_feat = x_chunk if self.cached_feat is None else torch.cat([self.cached_feat, x_chunk], dim=0)
        tail = self.remained_wav[FRAME_SHIFT * nf:]
        self.remained_wav = (tail * np.float32(gain)).astype(np.float32) if self._use_db else tail

        num_frames = int(self.cached_feat.shape[0])
        starts = chunk_starts(num_frames, is_end)
        if not starts:
            return None
        end = None
        for cur in starts:
            end = min(cur + DECODING_WINDOW, num_frames)
            out = eng.encode_chunk(self.cached_feat[cur:end], self._stream,
                                   required_cache_size=DECODING_CHUNK_SIZE * -1)
            if out is None:
                continue
            ids, maxp, _ = out
            if self._beam_conf is not None:
                # predict.py:320-322: beam_search_decoder.decode_chunk on this chunk's posteriors (state kept on the device)
                if self._sbeam is None:
                    from .engine import StreamBeam
                    self._sbeam = StreamBeam(eng, hotwords=self._hotwords, **self._beam_conf)
                rows = int(ids.shape[0])
                self._sbeam_result = self._sbeam.push(self._stream.last_logits, rows) if n_best is None else \
                    self._sbeam.push(self._stream.last_logits, rows, n_best=n_best)
                continue
            ids_h = ids.cpu().numpy()
            mp_h = maxp.cpu().numpy()
            self._hist_ids.extend(int(i) for i in ids_h)
            self._hist_probs.extend(mp_h[t] for t in range(len(ids_h)) if ids_h[t] != 0)
        self.cached_feat = self.cached_feat[end - CACHED_FEATURE_NUM:]
        vocab, dt = self._text_featurizer.vocab_list, ts.frame_seconds(eng)
        if self._beam_conf is not None:
            toks, score = self._sbeam_result[:2]
            if is_itn:
                raise Exception("masr_b200: inverse text normalisation (is_itn) is outside the hot-path scope")
            r = {'text': ids_to_text(toks, vocab), 'score': score}
            if timestamps:
                ts.beam_result(r, toks, self._sbeam.onsets() if toks else [], vocab, dt)
            if n_best is not None:
                hyps = self._sbeam_result[2] if len(self._sbeam_result) > 2 else [(toks, score)]
                r['n_best'] = nbest_dicts(hyps[:n_best], vocab)
            return r
        # greedy_decoder_chunk re-collapses the whole history (ctc_greedy_decoder.py:81-88)
        toks, prev = [], None
        for i in self._hist_ids:
            if i != prev and i != 0:
                toks.append(i)
            prev = i
        acc = np.float32(0.0)
        for p in self._hist_probs:
            acc = np.float32(acc + p)
        score = greedy_score(acc, len(self._hist_probs))
        text = ids_to_text(toks, vocab)
        if use_pun and is_end and len(text) > 0:
            logger.warning('标点符号模型没有初始化！')
        if is_itn:
            raise Exception("masr_b200: inverse text normalisation (is_itn) is outside the hot-path scope")
        r = {'text': text, 'score': score}
        return ts.greedy_result(r, self._hist_ids, vocab, dt) if timestamps else r

    def create_stream_pool(self, n_slots: int, max_frames: int = 3000, vad_model_path=None, vad_options=None,
                           timestamps=False, max_hotword_nodes: int = 0, n_best=None):
        """Additive: a ``StreamPool`` of ``n_slots`` concurrent streams over this predictor's model, decoding as the YAML
        says — greedy, or the GPU prefix beam search with the character or word LM this predictor loaded (if any).  Each slot's
        ``push`` results equal ``predict_stream`` on that stream alone.  ``max_frames``: encoder frames one stream may reach
        before it must be reset (40 ms each; 3000 = 2 minutes).

        ``vad_model_path`` (the silero VAD model file): instead a ``SegmentingStreamPool`` over that pool, which cuts every
        slot's live stream into utterances with ``GpuSileroVAD(vad_model_path, **vad_options)`` and decodes each one as a
        fresh ``predict_stream`` (masr_b200/segment_pool.py), so a stream may run for any length.

        ``timestamps``: every result also carries ``'tokens'`` (+ ``'words'``) as ``predict_stream(..., timestamps=True)``,
        timed since the slot's reset; with the VAD, segments and partials are timed since the slot's stream started.

        Hotwords: every slot boosts this predictor's list; ``max_hotword_nodes`` > 0 gives each slot room for its own list
        of up to that many automaton nodes (a list of n hotwords of k characters takes at most n * k + 1), set with
        ``set_hotwords(slot, hotwords)`` right after the slot's reset.

        ``n_best``: every result (with the VAD, every segment and partial) also carries ``'n_best'`` as in predict."""
        if not self.configs.streaming:
            raise Exception(f"不支持改该模型流式识别，当前模型：{self.configs.use_model}，参数streaming为：{self.configs.streaming}")
        from .stream_pool import StreamPool
        n_best = self._n_best(n_best)
        beam = self._beam_conf
        if beam is not None and (self._hotwords is not None or max_hotword_nodes > 0):
            beam = dict(beam, hotwords=self._hotwords, max_hotword_nodes=int(max_hotword_nodes))
        elif beam is None and max_hotword_nodes > 0:
            raise ValueError("hotwords need the prefix beam search (decoder: ctc_beam_search), not ctc_greedy")
        pool = StreamPool(self.predictor, self._text_featurizer.vocab_list, n_slots, use_db_normalization=self._use_db,
                          target_db=self._target_db, max_frames=max_frames, beam=beam, resample=self._resample,
                          timestamps=timestamps, hotword_score=self._hotword_score, n_best=n_best)
        if vad_model_path is None:
            return pool
        from .segment_pool import SegmentingStreamPool
        from .vad import GpuSileroVAD
        return SegmentingStreamPool(pool, GpuSileroVAD(vad_model_path, device=self.predictor.device, **(vad_options or {})))

    def reset_stream(self):
        """predict.py:346-353."""
        if self._stream is not None:
            self._stream.reset()
        self.remained_wav = None
        self.cached_feat = None
        self._hist_ids = []
        self._hist_probs = []
        if self._sbeam is not None:                          # predict.py:352-353: beam_search_decoder.reset_decoder()
            self._sbeam.reset()
        self._sbeam_result = ([], 0.0)


FRAME_SHIFT = 160
