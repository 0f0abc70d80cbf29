"""Freeze the reference's DeepSpeech2 outputs with ``encoder_conf.use_gru: True`` (GRU recurrences), on the CPU, through
``oracle/ref_shims.py``, at the shipped sizes (5 layers, rnn_size 1024):

    python tests/golden/make_deepspeech2_gru_golden.py [gru] [predictor_gru]

  * ``deepspeech2_gru_golden.npz``: the scripted model's ``get_encoder_out`` for a uni- and a bidirectional model (features,
    top-8 posteriors, frame ids, greedy text and score), and for the uni model a walk of ``get_encoder_out_chunk`` over
    67-frame windows at stride 64 that ends in a short window, carrying the state as inference_predictor.py:66-78 does
    (per-window top-8 posteriors and frame ids, and the h state after each window);
  * ``predictor_golden_deepspeech2_gru.json``: the real ``MASRPredictor`` (use_gpu=False, greedy) on an exported GRU model,
    whole utterance and PCM pushes.

Weights, CMVN, vocabulary and audio are regenerated from seeds by ``masr_b200.synth``; only the reference's outputs are stored.
"""
import json
import os
import sys
import tempfile

import numpy as np

from make_golden import HERE, V, make_audio, ref_shims, synth, torch, yaml

GRU_CASES = [  # (name, streaming, weight seed, audio kind, audio seed, samples)
    ("ds2gru_uni_speech_1p5s", True, 0, "speech", 45, 24000),
    ("ds2gru_bi_speech_1p2s", False, 1, "speech", 46, 19200 + 80),
]
# weight seed, audio kind, audio seed, samples: 281 feature frames = four full windows and a 25-frame one (5 encoder frames)
GRU_CHUNK_CASE = ("ds2gru_chunks", 0, "speech", 47, 160 * 280 + 400)
GRU_STREAM_CASE = ("ds2gru_stream_speech_3p75s", 0, "speech", 48, 60000, 8000)  # weight seed, kind, audio seed, samples, push


def reference_model(tmp, streaming, wseed):
    from masr.model_utils.deepspeech2.model import DeepSpeech2Model
    cfg = yaml.safe_load(open(os.path.join(ref_shims.REFERENCE_ROOT, "configs", "deepspeech2.yml"), encoding="utf-8"))
    cfg["encoder_conf"]["use_gru"] = True
    mi = os.path.join(tmp, f"mean_istd_{wseed}.json")
    synth.write_mean_istd(mi, wseed)
    model = DeepSpeech2Model(input_dim=80, vocab_size=V, mean_istd_path=mi, streaming=streaming,
                             encoder_conf=cfg["encoder_conf"], decoder_conf=cfg["decoder_conf"])
    model.load_state_dict(synth.to_torch(synth.deepspeech2_state_dict(wseed, V, streaming=streaming, use_gru=True)), strict=True)
    return model.eval(), cfg, mi


def gen_gru(tmp):
    from masr.data_utils.audio import AudioSegment
    from masr.data_utils.featurizer.audio_featurizer import AudioFeaturizer
    from masr.decoders.ctc_greedy_decoder import greedy_decoder
    af = AudioFeaturizer(feature_method="fbank", n_mels=80, sample_rate=16000, use_dB_normalization=True, target_dB=-20)
    vocab = synth.vocabulary(V)
    out, meta = {}, []
    for name, streaming, wseed, kind, aseed, n in GRU_CASES:
        scripted = reference_model(tmp, streaming, wseed)[0].export()
        x = make_audio(kind, aseed, n)
        feat = torch.from_numpy(af.featurize(AudioSegment.from_ndarray(x.copy(), 16000)))[None]
        with torch.no_grad():
            probs = scripted.get_encoder_out(feat, torch.tensor([feat.shape[1]]))[0]
        score, text = greedy_decoder(probs.numpy(), vocab)
        top = probs.topk(8, dim=1)
        out[name + "/feat"] = feat[0].numpy()
        out[name + "/top_p"] = top.values.numpy()
        out[name + "/top_i"] = top.indices.numpy().astype(np.int32)
        out[name + "/ids"] = probs.argmax(1).numpy().astype(np.int32)
        meta.append({"name": name, "streaming": streaming, "wseed": wseed, "kind": kind, "aseed": aseed, "samples": n,
                     "score": score, "text": text})
        print(name, "T", probs.shape[0], "score", score, "text", text)
    # chunk walk of the uni model: state carried window to window, as the reference predictor does
    name, wseed, kind, aseed, n = GRU_CHUNK_CASE
    scripted = reference_model(tmp, True, wseed)[0].export()
    feat = torch.from_numpy(af.featurize(AudioSegment.from_ndarray(make_audio(kind, aseed, n).copy(), 16000)))[None]
    h = c = torch.zeros([0, 0, 0, 0])
    starts, probs_l, h_l = [], [], []
    for cur in range(0, feat.shape[1] - 7 + 1, 64):
        x = feat[:, cur:cur + 67]
        with torch.no_grad():
            p, _, h, c = scripted.get_encoder_out_chunk(x, torch.tensor([x.shape[1]]), h, c)
        starts.append([cur, x.shape[1]])
        probs_l.append(p[0].numpy())
        h_l.append(h[:, 0, 0].numpy())                       # [layers, H] (forward only, batch 1)
    assert starts[-1][1] < 67
    out[name + "/feat"] = feat[0].numpy()
    out[name + "/windows"] = np.asarray(starts, np.int32)
    probs = torch.from_numpy(np.concatenate(probs_l))
    top = probs.topk(8, dim=1)
    out[name + "/top_p"] = top.values.numpy()
    out[name + "/top_i"] = top.indices.numpy().astype(np.int32)
    out[name + "/ids"] = probs.argmax(1).numpy().astype(np.int32)
    out[name + "/h"] = np.stack(h_l)
    meta.append({"name": name, "streaming": True, "wseed": wseed, "kind": kind, "aseed": aseed, "samples": n, "chunks": True})
    print(name, "windows", starts)
    out["meta"] = np.frombuffer(json.dumps(meta, ensure_ascii=False).encode("utf-8"), np.uint8)
    np.savez_compressed(os.path.join(HERE, "deepspeech2_gru_golden.npz"), **out)


def gen_predictor_gru(tmp):
    """The real ``MASRPredictor`` with a streaming GRU DeepSpeech2, greedy: whole utterance and PCM pushes."""
    from masr.predict import MASRPredictor
    name, wseed, kind, aseed, n, push = GRU_STREAM_CASE
    model, cfg, mi = reference_model(tmp, True, wseed)
    mp = os.path.join(tmp, "inference_ds2gru.pt")
    torch.jit.save(model.export(), mp)
    vp = os.path.join(tmp, "vocabulary.txt")
    synth.write_vocabulary(vp, V)
    cfg["dataset_conf"]["dataset_vocab"] = vp
    cfg["dataset_conf"]["mean_istd_path"] = mi
    cfg["decoder"] = "ctc_greedy"
    cfg["streaming"] = True
    np.random.seed(0)
    pred = MASRPredictor(configs=cfg, model_path=mp, use_gpu=False)
    x = make_audio(kind, aseed, n)
    whole = pred.predict(audio_data=x.copy())
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    pushes = []
    pred.reset_stream()
    for s in range(0, len(pcm), push):
        r = pred.predict_stream(audio_data=pcm[s:s + push].tobytes(), is_end=s + push >= len(pcm))
        pushes.append(None if r is None else {"text": r["text"], "score": r["score"]})
    pred.reset_stream()
    data = {"name": name, "wseed": wseed, "kind": kind, "aseed": aseed, "samples": n, "push": push,
            "whole": whole, "pushes_pcm": pushes}
    with open(os.path.join(HERE, "predictor_golden_deepspeech2_gru.json"), "w", encoding="utf-8") as f:
        json.dump(data, f, ensure_ascii=False, indent=1)
    print("deepspeech2 gru predictor whole", whole)
    print("pushes", pushes)


if __name__ == "__main__":
    torch.set_num_threads(8)
    with tempfile.TemporaryDirectory() as tmp:
        which = sys.argv[1:] or ["gru", "predictor_gru"]
        if "gru" in which:
            gen_gru(tmp)
        if "predictor_gru" in which:
            gen_predictor_gru(tmp)
