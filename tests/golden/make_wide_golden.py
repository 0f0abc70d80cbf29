"""Freeze the reference's outputs for the wide Conformer (``output_size: 512``, ``attention_heads: 8``, the other size
configs/conformer.yml names) by running the UNMODIFIED reference in the build container through ``oracle/ref_shims.py``:

    python tests/golden/make_wide_golden.py       # rewrites conformer_wide_golden.npz, predictor_golden_wide.json

  * ``conformer_wide_golden.npz``: features, encoder output, frame ids, top-8 posteriors, text and score of the exported
    (TorchScript) model for a few short utterances, causal and non-causal;
  * ``predictor_golden_wide.json``: the real ``MASRPredictor`` (use_gpu=False, greedy) on the exported causal model: the
    whole-utterance result and every ``predict_stream`` push.

The weights are ``synth.conformer_state_dict(seed, output_size=512, attention_heads=8)``, so only outputs are stored.
"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))

from oracle import ref_shims  # noqa: E402

ref_shims.install()

import torch  # noqa: E402
import yaml  # noqa: E402

from masr_b200 import synth  # noqa: E402

V = synth.DEFAULT_VOCAB_SIZE
WIDE = {"output_size": 512, "attention_heads": 8}

ENCODER_CASES = [  # (name, streaming, weight seed, audio kind, audio seed, samples)
    ("wide_causal_speech_2p5s", True, 0, "speech", 50, 40000),
    ("wide_causal_noise_2s", True, 0, "noise", 51, 32000 + 55),
    ("wide_noncausal_speech_3s", False, 1, "speech", 52, 48000),
]
STREAM_CASE = ("wide_stream_speech_3p5s", 0, "speech", 53, 56000 + 91, 8000)  # weight seed, kind, audio seed, samples, push


def make_audio(kind, seed, n):
    return synth.noise_audio(seed, n) if kind == "noise" else synth.speechlike_audio(seed, n)


def build_reference_model(tmp, streaming, wseed):
    from masr.model_utils.conformer.model import ConformerModel
    cfg = yaml.safe_load(open(os.path.join(ref_shims.REFERENCE_ROOT, "configs", "conformer.yml"), encoding="utf-8"))
    cfg["encoder_conf"].update(WIDE)
    mi = os.path.join(tmp, f"mean_istd_{wseed}.json")
    synth.write_mean_istd(mi, wseed)
    model = ConformerModel(input_dim=80, vocab_size=V, mean_istd_path=mi, streaming=streaming,
                           encoder_conf=cfg["encoder_conf"], decoder_conf=cfg["decoder_conf"], **cfg["model_conf"])
    sd = synth.to_torch(synth.conformer_state_dict(wseed, V, **WIDE))
    res = model.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.startswith("decoder.") for k in res.missing_keys)
    return model.eval(), cfg, mi


def gen_encoder(tmp):
    from masr.data_utils.audio import AudioSegment
    from masr.data_utils.featurizer.audio_featurizer import AudioFeaturizer
    from masr.decoders.ctc_greedy_decoder import greedy_decoder
    af = AudioFeaturizer(feature_method="fbank", n_mels=80, sample_rate=16000, use_dB_normalization=True, target_dB=-20)
    vocab = synth.vocabulary(V)
    out, meta = {}, []
    for name, streaming, wseed, kind, aseed, n in ENCODER_CASES:
        model, _, _ = build_reference_model(tmp, streaming, wseed)
        scripted = model.export()
        x = make_audio(kind, aseed, n)
        feat = torch.from_numpy(af.featurize(AudioSegment.from_ndarray(x.copy(), 16000)))[None]
        with torch.no_grad():
            probs = scripted.get_encoder_out(feat, torch.tensor([feat.shape[1]]))[0]
            enc, _ = model.encoder(feat, torch.tensor([feat.shape[1]]), decoding_chunk_size=-1, num_decoding_left_chunks=-1)
        score, text = greedy_decoder(probs.numpy(), vocab)
        top = probs.topk(8, dim=1)
        out[name + "/feat"] = feat[0].numpy()
        out[name + "/enc"] = enc[0].numpy()
        out[name + "/top_p"] = top.values.numpy()
        out[name + "/top_i"] = top.indices.numpy().astype(np.int32)
        out[name + "/ids"] = probs.argmax(1).numpy().astype(np.int32)
        meta.append({"name": name, "streaming": streaming, "wseed": wseed, "kind": kind, "aseed": aseed, "samples": n,
                     "score": score, "text": text})
        print(name, "T", probs.shape[0], "score", score, "text", text)
    out["meta"] = np.frombuffer(json.dumps(meta, ensure_ascii=False).encode("utf-8"), np.uint8)
    np.savez_compressed(os.path.join(HERE, "conformer_wide_golden.npz"), **out)


def gen_predictor(tmp):
    from masr.predict import MASRPredictor
    name, wseed, kind, aseed, n, push = STREAM_CASE
    model, cfg, mi = build_reference_model(tmp, True, wseed)
    mp = os.path.join(tmp, "inference.pt")
    torch.jit.save(model.export(), mp)
    vp = os.path.join(tmp, "vocabulary.txt")
    synth.write_vocabulary(vp, V)
    cfg["dataset_conf"]["dataset_vocab"] = vp
    cfg["dataset_conf"]["mean_istd_path"] = mi
    cfg["decoder"] = "ctc_greedy"
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
            "output_size": WIDE["output_size"], "attention_heads": WIDE["attention_heads"],
            "whole": whole, "pushes_pcm": pushes}
    with open(os.path.join(HERE, "predictor_golden_wide.json"), "w", encoding="utf-8") as f:
        json.dump(data, f, ensure_ascii=False, indent=1)
    print("wide predictor whole", whole)
    print("pushes", pushes)


if __name__ == "__main__":
    torch.set_num_threads(8)
    with tempfile.TemporaryDirectory() as tmp:
        gen_encoder(tmp)
        gen_predictor(tmp)
