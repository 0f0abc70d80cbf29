"""Freeze the reference's DeepSpeech2 outputs at ``encoder_conf.rnn_size: 2048`` (the large-data size of
configs/deepspeech2.yml), LSTM and GRU, on the CPU, through ``oracle/ref_shims.py``:

    python tests/golden/make_wide_deepspeech2_golden.py [model] [predictor]

  * ``deepspeech2_wide_golden.npz``: per cell, the scripted model's ``get_encoder_out`` for a uni- and a bidirectional model
    (features, top-8 posteriors, frame ids, greedy text and score), and for the uni model a walk of
    ``get_encoder_out_chunk`` over 67-frame windows at stride 64 that ends in a short window, carrying the state as
    inference_predictor.py:66-78 does (per-window top-8 posteriors and frame ids, the h state after each window and, for
    the LSTM, the c state);
  * ``predictor_golden_deepspeech2_wide.json``: per cell, the real ``MASRPredictor`` (use_gpu=False, greedy) on an exported
    streaming model, whole utterance and PCM pushes.

Weights, CMVN, vocabulary and audio are regenerated from seeds by ``masr_b200.synth``; only the reference's outputs are stored.
"""
import json
import os
import sys
import tempfile

import numpy as np

from make_golden import HERE, V, make_audio, ref_shims, synth, torch, yaml

HIDDEN = 2048
CELLS = ("lstm", "gru")
# weight seed per (cell, streaming): the streaming GRU of seed 0 decodes these utterances to all blanks, seed 2 does not
WSEED = {("lstm", True): 0, ("gru", True): 2, ("lstm", False): 1, ("gru", False): 1}
WIDE_CASES = [  # (tag, streaming, audio kind, audio seed, samples)
    ("uni_speech_1p5s", True, "speech", 55, 24000),
    ("bi_speech_1p2s", False, "speech", 56, 19200 + 80),
]
# audio kind, audio seed, samples: 281 feature frames = four full windows and a 25-frame one (5 encoder frames)
WIDE_CHUNK_CASE = ("chunks", "speech", 57, 160 * 280 + 400)
WIDE_STREAM_CASE = ("stream_speech_3p75s", "speech", 58, 60000, 8000)  # kind, audio seed, samples, push


def reference_model(tmp, cell, streaming, wseed):
    from masr.model_utils.deepspeech2.model import DeepSpeech2Model
    cfg = yaml.safe_load(open(os.path.join(ref_shims.REFERENCE_ROOT, "configs", "deepspeech2.yml"), encoding="utf-8"))
    cfg["encoder_conf"]["rnn_size"] = HIDDEN
    cfg["encoder_conf"]["use_gru"] = cell == "gru"
    mi = os.path.join(tmp, f"mean_istd_{wseed}.json")
    synth.write_mean_istd(mi, wseed)
    model = DeepSpeech2Model(input_dim=80, vocab_size=V, mean_istd_path=mi, streaming=streaming,
                             encoder_conf=cfg["encoder_conf"], decoder_conf=cfg["decoder_conf"])
    sd = synth.deepspeech2_state_dict(wseed, V, streaming=streaming, hidden=HIDDEN, use_gru=cell == "gru")
    model.load_state_dict(synth.to_torch(sd), strict=True)
    return model.eval(), cfg, mi


def _top(out, key, probs):
    top = probs.topk(8, dim=1)
    out[key + "/top_p"] = top.values.numpy()
    out[key + "/top_i"] = top.indices.numpy().astype(np.int32)
    out[key + "/ids"] = probs.argmax(1).numpy().astype(np.int32)


def gen_model(tmp):
    from masr.data_utils.audio import AudioSegment
    from masr.data_utils.featurizer.audio_featurizer import AudioFeaturizer
    from masr.decoders.ctc_greedy_decoder import greedy_decoder
    af = AudioFeaturizer(feature_method="fbank", n_mels=80, sample_rate=16000, use_dB_normalization=True, target_dB=-20)
    vocab = synth.vocabulary(V)
    out, meta = {}, []
    for cell in CELLS:
        for tag, streaming, kind, aseed, n in WIDE_CASES:
            name = f"ds2wide_{cell}_{tag}"
            wseed = WSEED[cell, streaming]
            scripted = reference_model(tmp, cell, streaming, wseed)[0].export()
            x = make_audio(kind, aseed, n)
            feat = torch.from_numpy(af.featurize(AudioSegment.from_ndarray(x.copy(), 16000)))[None]
            with torch.no_grad():
                probs = scripted.get_encoder_out(feat, torch.tensor([feat.shape[1]]))[0]
            score, text = greedy_decoder(probs.numpy(), vocab)
            out[name + "/feat"] = feat[0].numpy()
            _top(out, name, probs)
            meta.append({"name": name, "cell": cell, "streaming": streaming, "wseed": wseed, "kind": kind, "aseed": aseed,
                         "samples": n, "score": score, "text": text})
            print(name, "T", probs.shape[0], "score", score, "text", text)
            del scripted
        # chunk walk of the uni model: state carried window to window, as the reference predictor does
        tag, kind, aseed, n = WIDE_CHUNK_CASE
        name = f"ds2wide_{cell}_{tag}"
        wseed = WSEED[cell, True]
        scripted = reference_model(tmp, cell, True, wseed)[0].export()
        feat = torch.from_numpy(af.featurize(AudioSegment.from_ndarray(make_audio(kind, aseed, n).copy(), 16000)))[None]
        h = c = torch.zeros([0, 0, 0, 0])
        starts, probs_l, h_l, c_l = [], [], [], []
        for cur in range(0, feat.shape[1] - 7 + 1, 64):
            x = feat[:, cur:cur + 67]
            with torch.no_grad():
                p, _, h, c = scripted.get_encoder_out_chunk(x, torch.tensor([x.shape[1]]), h, c)
            starts.append([cur, x.shape[1]])
            probs_l.append(p[0].numpy())
            h_l.append(h.reshape(-1, HIDDEN).numpy().copy())    # [layers, H] (forward only, batch 1)
            c_l.append(c.reshape(-1, HIDDEN).numpy().copy())
        assert starts[-1][1] < 67 and h_l[0].shape == (5, HIDDEN)
        out[name + "/feat"] = feat[0].numpy()
        out[name + "/windows"] = np.asarray(starts, np.int32)
        _top(out, name, torch.from_numpy(np.concatenate(probs_l)))
        out[name + "/h"] = np.stack(h_l)
        if cell == "lstm":
            out[name + "/c"] = np.stack(c_l)
        meta.append({"name": name, "cell": cell, "streaming": True, "wseed": wseed, "kind": kind, "aseed": aseed,
                     "samples": n, "chunks": True})
        print(name, "windows", starts)
        del scripted
    out["meta"] = np.frombuffer(json.dumps(meta, ensure_ascii=False).encode("utf-8"), np.uint8)
    np.savez_compressed(os.path.join(HERE, "deepspeech2_wide_golden.npz"), **out)


def gen_predictor(tmp):
    """The real ``MASRPredictor`` with a streaming 2048-wide DeepSpeech2 of either cell, greedy: whole utterance and PCM
    pushes."""
    from masr.predict import MASRPredictor
    tag, kind, aseed, n, push = WIDE_STREAM_CASE
    data = {"name": tag, "hidden": HIDDEN, "kind": kind, "aseed": aseed, "samples": n, "push": push}
    for cell in CELLS:
        wseed = WSEED[cell, True]
        model, cfg, mi = reference_model(tmp, cell, True, wseed)
        mp = os.path.join(tmp, f"inference_ds2wide_{cell}.pt")
        torch.jit.save(model.export(), mp)
        del model
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
        data[cell] = {"wseed": wseed, "whole": whole, "pushes_pcm": pushes}
        print(f"deepspeech2 wide {cell} predictor whole", whole)
        print("pushes", pushes)
        del pred
        os.remove(mp)
    with open(os.path.join(HERE, "predictor_golden_deepspeech2_wide.json"), "w", encoding="utf-8") as f:
        json.dump(data, f, ensure_ascii=False, indent=1)


if __name__ == "__main__":
    torch.set_num_threads(8)
    with tempfile.TemporaryDirectory() as tmp:
        which = sys.argv[1:] or ["model", "predictor"]
        if "model" in which:
            gen_model(tmp)
        if "predictor" in which:
            gen_predictor(tmp)
