"""Freeze what tests/test_oracle_vs_reference.py compares the oracle against: the UNMODIFIED reference's featurizer outputs,
its full-utterance encoder output and its chunk-by-chunk outputs and caches (Conformer, Squeezeformer, Efficient Conformer,
DeepSpeech2), run through ``oracle/ref_shims.py`` on the seeded synthetic inputs of that test.

    python tests/golden/make_reference_chunks.py      # rewrites tests/golden/reference_chunks_golden.npz

Large tensors are stored as a fixed, seeded sample of elements (flat index, value) plus the per-frame argmax of
probabilities, so the file stays small; ``sampled()`` in the test reads them back.
"""
import os
import sys
import tempfile
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "reference_chunks_golden.npz")
SAMPLE = 1024


def sample_index(name, n):
    """The element sample of tensor `name` (n elements): fixed by the name, shared with the test."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    return np.sort(rng.choice(n, size=min(n, SAMPLE), replace=False)).astype(np.int64)


def put(store, name, t, argmax=False, full=False):
    a = np.asarray(t.detach().cpu().numpy() if hasattr(t, "detach") else t, dtype=np.float32)
    store[name + ".shape"] = np.array(a.shape, dtype=np.int64)
    if full:
        store[name] = a
        return
    store[name + ".val"] = a.reshape(-1)[sample_index(name, a.size)]
    if argmax:
        store[name + ".argmax"] = a.argmax(-1).astype(np.int32)


def main():
    import torch
    import yaml
    from conftest import make_audio, synth_weights
    from masr_b200 import synth
    from oracle import fbank as ob, ref_shims
    ref_shims.install()
    from masr.data_utils.audio import AudioSegment
    from masr.data_utils.featurizer.audio_featurizer import AudioFeaturizer
    store = {}
    af = AudioFeaturizer(feature_method="fbank", n_mels=80, sample_rate=16000, use_dB_normalization=True, target_dB=-20)
    for kind, seed, n in [("noise", 5, 20000), ("speech", 6, 33333)]:
        put(store, f"fbank.{kind}{seed}", af.featurize(AudioSegment.from_ndarray(make_audio(kind, seed, n).copy(), 16000)), full=True)
    pcm = (make_audio("speech", 7, 8000) * 20000).astype(np.int16)
    put(store, "fbank.pcm7", af.featurize(AudioSegment.from_pcm_bytes(pcm.tobytes())), full=True)

    def model(cls, yml, sd, strict=False, **kw):
        cfg_y = yaml.safe_load(open(os.path.join(ref_shims.REFERENCE_ROOT, "configs", yml), encoding="utf-8"))
        with tempfile.TemporaryDirectory() as tmp:
            mi = os.path.join(tmp, "mi.json")
            synth.write_mean_istd(mi, 0)
            m = cls(input_dim=80, vocab_size=synth.DEFAULT_VOCAB_SIZE, mean_istd_path=mi, streaming=True,
                    encoder_conf=cfg_y["encoder_conf"], decoder_conf=cfg_y["decoder_conf"], **kw).eval()
        m.load_state_dict(synth.to_torch(sd), strict=strict)
        return m

    def chunks(prefix, m, feat, lens=False):
        att = torch.zeros(0, 0, 0, 0)
        cnn = torch.zeros(0, 0, 0, 0)
        off, i, nf = 0, 0, feat.shape[1]
        step_min = 67 if prefix == "conformer" else 7
        for cur in range(0, nf - step_min + 1, 64):
            ch = feat[:, cur:min(cur + 67, nf)]
            if lens:
                pr, ln, att, cnn = m.get_encoder_out_chunk(ch, torch.tensor([ch.shape[1]]), att, cnn)
                store[f"{prefix}.{i}.lens"] = np.array([int(ln[0])], dtype=np.int64)
                pr = pr[0]
            else:
                pr, att, cnn = m.get_encoder_out_chunk(ch, off, -16, att, cnn)
                off += pr.shape[1]
            put(store, f"{prefix}.{i}.probs", pr, argmax=True)
            put(store, f"{prefix}.{i}.att", att)
            put(store, f"{prefix}.{i}.cnn", cnn)
            i += 1
        store[f"{prefix}.chunks"] = np.array([i], dtype=np.int64)

    cfg_c = yaml.safe_load(open(os.path.join(ref_shims.REFERENCE_ROOT, "configs", "conformer.yml"), encoding="utf-8"))
    from masr.model_utils.conformer.model import ConformerModel
    with torch.no_grad():
        m = model(ConformerModel, "conformer.yml", synth_weights(0), **cfg_c["model_conf"])
        feat = torch.from_numpy(ob.featurize(make_audio("speech", 8, 16000 * 3)))[None]
        put(store, "conformer.full", m.get_encoder_out(feat, torch.tensor([feat.shape[1]])), argmax=True)
        chunks("conformer", m, feat)

        from masr.model_utils.squeezeformer.model import SqueezeformerModel
        cfg_s = yaml.safe_load(open(os.path.join(ref_shims.REFERENCE_ROOT, "configs", "squeezeformer.yml"), encoding="utf-8"))
        m = model(SqueezeformerModel, "squeezeformer.yml", synth.squeezeformer_state_dict(0, streaming=True), **cfg_s["model_conf"])
        chunks("squeezeformer", m, torch.from_numpy(ob.featurize(make_audio("speech", 9, 16000 * 3 + 4000)))[None])

        from masr.model_utils.efficient_conformer.model import EfficientConformerModel
        cfg_e = yaml.safe_load(open(os.path.join(ref_shims.REFERENCE_ROOT, "configs", "efficient_conformer.yml"), encoding="utf-8"))
        m = model(EfficientConformerModel, "efficient_conformer.yml", synth.efficient_conformer_state_dict(0), **cfg_e["model_conf"])
        chunks("efficient", m, torch.from_numpy(ob.featurize(make_audio("speech", 13, 16000 * 3 + 4000)))[None])

        from masr.model_utils.deepspeech2.model import DeepSpeech2Model
        m = model(DeepSpeech2Model, "deepspeech2.yml", synth.deepspeech2_state_dict(0, streaming=True), strict=True)
        chunks("deepspeech2", m, torch.from_numpy(ob.featurize(make_audio("speech", 14, 16000 * 3 + 4000)))[None], lens=True)
    np.savez_compressed(OUT, **store)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
