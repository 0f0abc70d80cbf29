"""Dev tool: end-to-end throughput (host float32 waveforms in, token ids + scores out, one blocking call per batch) of the
per-GPU shard of every BASELINE.json config that is not the headline — one JSON line each.  Synthetic audio + weights.
    config 2  conformer.yml streaming=False, 32 x 10 s, ctc_greedy
    config 4  efficient_conformer.yml streaming=False, 32 x 10 s per GPU (256 over 8), ctc_beam_search (no LM)
    config 5  conformer.yml (streaming-trained), 64 utterances of 1-30 s per GPU (512 over 8), ctc_beam_search (no LM)
    config 4lm / 4plm / 5lm  the same beam-search configs with a synthetic character 5-gram ARPA LM (alpha 2.2, beta 4.3, the
              shipped configs' values; a few million n-grams, generated into a temporary directory on first use)
    plus      squeezeformer.yml / deepspeech2.yml whole-utterance, 32 x 10 s, ctc_greedy; deepspeech2gru the same with
              encoder_conf.use_gru: True (GRU recurrences); deepspeech2wide: rnn_size 2048, LSTM and GRU, uni and bi
Numbers printed here are dev measurements (CUDA-synchronised wall clock around the public engine call), not bench values."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from masr_b200 import synth
from masr_b200.deepspeech2 import DeepSpeech2Engine
from masr_b200.engine import ConformerEngine, EfficientConformerEngine
from masr_b200.squeezeformer import SqueezeformerEngine

BEAM = dict(beam_size=300, cutoff_prob=0.99, cutoff_top_n=40)
only = set(sys.argv[1:])


def run(name, eng, waves, fn, reps=5, oracle=None, sample=(0,)):
    """oracle(wave) -> expected greedy token ids of one utterance on the CPU (the oracle port): the timed call's output is
    checked against it on `sample` before the timing (VERDICT r1: the config lines carried no correctness check)."""
    if only and name.split()[0] not in only:
        return
    for _ in range(2):
        out = fn(waves)
    verified = None
    if oracle is not None:
        toks = out.tokens if hasattr(out, "tokens") else out[0]
        verified = all(list(toks[i]) == list(oracle(waves[i])) for i in sample)
        assert verified, f"{name}: token ids differ from the CPU oracle"
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn(waves)
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / reps
    audio = sum(len(w) for w in waves) / 16000.0
    print(json.dumps({"config": name, "utterances": len(waves), "audio_s": audio, "ms_per_batch": dt * 1e3,
                      "audio_seconds_per_second": audio / dt,
                      "ids_match_cpu_oracle_on_sample": None if verified is None else {"utterances": list(sample), "ok": verified}}), flush=True)


def beam_kernel_ms(name, eng, waves, fn, reps=3):
    """Event-timed prefix_beam kernel time of one blocking call (the engine's per-kernel profile)."""
    if only and name.split()[0] not in only:
        return
    fn(waves)
    eng.profile(True)
    for _ in range(reps):
        fn(waves)
    torch.cuda.synchronize()
    n, ms = eng.profile_summary()["prefix_beam"]
    eng.profile(False)
    print(json.dumps({"config": name, "prefix_beam_kernel_ms": ms / reps}), flush=True)


_LM = []


def big_lm():
    """The synthetic 5-gram (3000 characters, 200k sentences): loaded once, with its size and host load time printed."""
    if not _LM:
        import tempfile
        from masr_b200.lm import CharLM
        d = tempfile.mkdtemp(prefix="masr_lm_")
        p = os.path.join(d, "char5.arpa")
        t0 = time.perf_counter()
        synth.character_lm_arpa(p, seed=5, order=5, n_chars=3000, n_sentences=200000)
        t_gen = time.perf_counter() - t0
        lm = CharLM(p, synth.vocabulary())
        print(json.dumps({"lm": "synthetic character 5-gram", "arpa_bytes": os.path.getsize(p), "ngrams": lm.read_counts,
                          "kept": lm.kept_counts, "table_bytes": lm.table_bytes, "load_cpu_s": lm.load_seconds,
                          "generate_s": t_gen}), flush=True)
        os.remove(p)
        os.rmdir(d)
        _LM.append(lm)
    return _LM[0]


def want(*names):
    return not only or bool(only & set(names))


LMW = dict(alpha=2.2, beta=4.3)


def greedy_oracle(mod, sd, cfg, batched=True):
    from oracle import ctc as octc, fbank as ob

    def f(w):
        with torch.no_grad():
            feat = torch.from_numpy(ob.featurize(w.copy()))
            probs = mod.get_encoder_out(sd, cfg, feat[None] if batched else feat)[0].numpy()
        return octc.collapse(octc.best_path(probs)[0])
    return f


from oracle import conformer as oc, deepspeech2 as ods, deepspeech2_gru as odg, efficient_conformer as oe, squeezeformer as osq  # noqa: E402

tens = [synth.noise_audio(1000 + i, 160000) for i in range(32)]
rng = np.random.default_rng(0)
varlen = [synth.noise_audio(2000 + i, int(n)) for i, n in enumerate(rng.integers(16000, 480001, 64))]

sdn = synth.conformer_state_dict(0)
e = ConformerEngine(sdn, streaming=False)
run("config2 conformer.yml streaming=False 32x10s ctc_greedy", e, tens, lambda w: e.transcribe(w),
    oracle=greedy_oracle(oc, synth.to_torch(sdn), oc.ConformerConfig(causal=False)), sample=(0, 31))
del e
sdn = synth.efficient_conformer_state_dict(0)
e = EfficientConformerEngine(sdn, streaming=False)
run("config4 efficient_conformer.yml streaming=False 32x10s/GPU ctc_beam_search(300,40,0.99,no LM)", e, tens, lambda w: e.transcribe_beam(w, **BEAM))
beam_kernel_ms("config4 prefix beam kernel, no LM", e, tens, lambda w: e.transcribe_beam(w, **BEAM))
if want("config4lm", "config4plm"):
    lm = big_lm()
    run("config4lm efficient_conformer.yml streaming=False 32x10s/GPU ctc_beam_search(300,40,0.99, char 5-gram LM)", e, tens,
        lambda w: e.transcribe_beam(w, **BEAM, lm=lm, **LMW))
    beam_kernel_ms("config4lm prefix beam kernel, char 5-gram LM", e, tens, lambda w: e.transcribe_beam(w, **BEAM, lm=lm, **LMW))
def piped(w, e_=None):
    return list(e.transcribe_beam_pipelined([w] * 4, **BEAM))[-1]


if not only or "config4p" in only:
    # throughput form of config 4: a stream of batches, the beam search of batch k under the encoder of batch k+1
    for _ in range(2):
        piped(tens)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    n_b = 12
    res = list(e.transcribe_beam_pipelined([tens] * n_b, **BEAM))
    torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / n_b
    same = res[-1][0] == e.transcribe_beam(tens, **BEAM)[0]
    assert same
    print(json.dumps({"config": "config4p efficient_conformer.yml streaming=False 32x10s/GPU ctc_beam_search, PIPELINED stream of batches (beam search of batch k on a second stream under the encoder of batch k+1)",
                      "utterances": 32, "audio_s": 320.0, "ms_per_batch": dt * 1e3, "audio_seconds_per_second": 320.0 / dt,
                      "equals_blocking_call": bool(same)}), flush=True)
if want("config4plm"):
    lm = big_lm()
    torch.cuda.synchronize(); t0 = time.perf_counter()
    n_b = 12
    res = list(e.transcribe_beam_pipelined([tens] * n_b, **BEAM, lm=lm, **LMW))
    torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / n_b
    same = res[-1] == e.transcribe_beam(tens, **BEAM, lm=lm, **LMW)
    assert same
    print(json.dumps({"config": "config4plm efficient_conformer.yml 32x10s/GPU ctc_beam_search + char 5-gram LM, PIPELINED stream of batches",
                      "utterances": 32, "audio_s": 320.0, "ms_per_batch": dt * 1e3, "audio_seconds_per_second": 320.0 / dt,
                      "equals_blocking_call": bool(same)}), flush=True)
run("config4g efficient_conformer.yml streaming=False 32x10s/GPU ctc_greedy", e, tens, lambda w: e.transcribe(w),
    oracle=greedy_oracle(oe, synth.to_torch(sdn), oe.EfficientConfig(causal=False)), sample=(0, 31))
del e
sdn = synth.conformer_state_dict(0)
e = ConformerEngine(sdn, streaming=True)
run("config5 conformer.yml streaming-trained 64 x 1-30s/GPU ctc_beam_search(300,40,0.99,no LM)", e, varlen, lambda w: e.transcribe_beam(w, **BEAM), reps=3)
beam_kernel_ms("config5 prefix beam kernel, no LM", e, varlen, lambda w: e.transcribe_beam(w, **BEAM))
if want("config5lm"):
    lm = big_lm()
    run("config5lm conformer.yml streaming-trained 64 x 1-30s/GPU ctc_beam_search(300,40,0.99, char 5-gram LM)", e, varlen,
        lambda w: e.transcribe_beam(w, **BEAM, lm=lm, **LMW), reps=3)
    beam_kernel_ms("config5lm prefix beam kernel, char 5-gram LM", e, varlen, lambda w: e.transcribe_beam(w, **BEAM, lm=lm, **LMW))
run("config5g conformer.yml streaming-trained 64 x 1-30s/GPU ctc_greedy", e, varlen, lambda w: e.transcribe(w), reps=3,
    oracle=greedy_oracle(oc, synth.to_torch(sdn), oc.ConformerConfig()), sample=(int(np.argmin([len(w) for w in varlen])), 5))
del e
sdn = synth.squeezeformer_state_dict(0, streaming=True)
e = SqueezeformerEngine(sdn, streaming=True)
run("squeezeformer squeezeformer.yml 32x10s ctc_greedy (whole utterance)", e, tens, lambda w: e.transcribe(w),
    oracle=greedy_oracle(osq, synth.to_torch(sdn), osq.SqueezeformerConfig(causal=True)), sample=(0,))
del e
sdn = synth.deepspeech2_state_dict(0)
e = DeepSpeech2Engine(sdn, streaming=True)
run("deepspeech2 deepspeech2.yml 32x10s ctc_greedy (whole utterance)", e, tens, lambda w: e.transcribe(w),
    oracle=greedy_oracle(ods, synth.to_torch(sdn), ods.DS2Config()), sample=(0,))
del e
sdn = synth.deepspeech2_state_dict(0, use_gru=True)
e = DeepSpeech2Engine(sdn, streaming=True)
run("deepspeech2gru deepspeech2.yml use_gru=True 32x10s ctc_greedy (whole utterance)", e, tens, lambda w: e.transcribe(w),
    oracle=greedy_oracle(odg, synth.to_torch(sdn), ods.DS2Config()), sample=(0,))
for use_gru in (False, True):         # encoder_conf.rnn_size: 2048 (tensor-core persistent recurrence), uni and bi
    for streaming in (True, False):
        if not want("deepspeech2wide"):
            break
        del e
        torch.cuda.empty_cache()
        sdn = synth.deepspeech2_state_dict(0, streaming=streaming, hidden=2048, use_gru=use_gru)
        e = DeepSpeech2Engine(sdn, streaming=streaming)
        run(f"deepspeech2wide deepspeech2.yml rnn_size=2048 use_gru={use_gru} streaming={streaming} 32x10s ctc_greedy "
            "(whole utterance)", e, tens, lambda w: e.transcribe(w), reps=3,
            oracle=greedy_oracle(odg if use_gru else ods, synth.to_torch(sdn), ods.DS2Config(hidden=2048, bidirectional=not streaming)),
            sample=(0,))
