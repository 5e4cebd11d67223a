"""Generate tests/golden/wav2vec_tiny.npz by running the REAL reference wav2vec2 feature extractor on CPU.

Runs only where the reference tree exists (it is not needed anywhere else); its output is committed and pins
oracle/wav2vec2_oracle.py to the reference's behaviour (tests/test_audio_cpu.py).  Nothing from the reference is copied
into this repository: its modules are loaded, and two of its functions compiled, from the reference files in place.

usage:  python tests/golden/make_golden_audio.py [--ref /root/reference]
"""
import argparse
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def golden_audio(ref_root):
    """wav2vec2 feature extractor on a tiny config: the reference's own Wav2Vec2Model subclass
    (utils/src/audio_analysis/wav2vec2.py, with torch_utils.py's linear_interpolation) and the bodies of its get_embedding
    (utils/audio_process.py:18-41) and SVITalkVideoPipeline.get_audio_embedding (diffsynth/pipelines/svi_video_talk.py:412-430).
    The two modules are loaded by file path under temporary names (the reference's top-level `utils` package would clash
    with this repository's); the two functions are compiled out of the reference files with ast, with the librosa /
    pyloudnorm step replaced by the synthetic 16 kHz waveform — nothing is copied into this repository."""
    import ast
    import importlib.util
    from transformers import Wav2Vec2Config, Wav2Vec2FeatureExtractor
    from tools import synth_audio as SA
    names = ("utils", "utils.src", "utils.src.audio_analysis", "utils.src.audio_analysis.torch_utils")
    saved = {n: sys.modules.get(n) for n in names}
    try:
        for n in names[:3]:
            m = types.ModuleType(n)
            m.__path__ = []
            sys.modules[n] = m
        base = os.path.join(ref_root, "utils", "src", "audio_analysis")
        spec = importlib.util.spec_from_file_location("utils.src.audio_analysis.torch_utils", os.path.join(base, "torch_utils.py"))
        tu = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = tu
        spec.loader.exec_module(tu)
        spec = importlib.util.spec_from_file_location("_ref_wav2vec2", os.path.join(base, "wav2vec2.py"))
        w2v = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = w2v                                  # transformers looks its model classes up there
        spec.loader.exec_module(w2v)
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m

    def compiled(path, name, ns):
        tree = ast.parse(open(path).read())
        nodes = [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == name]
        exec(compile(ast.Module(body=[nodes[0]], type_ignores=[]), path, "exec"), ns)
        return ns[name]

    from einops import rearrange
    cfg = SA.TINY
    conf = Wav2Vec2Config(**cfg, attn_implementation="eager")        # the subclass sets output_attentions, refused under SDPA
    model = w2v.Wav2Vec2Model(conf).eval()
    sd = SA.make_state_dict(cfg, seed=0)
    model.load_state_dict(sd, strict=True)
    fe = Wav2Vec2FeatureExtractor(**{k: v for k, v in SA.PREPROCESSOR.items()})
    speech = SA.make_waveform(6.0, seed=0)                              # 16 kHz mono; T = 150 video frames
    get_embedding = compiled(os.path.join(ref_root, "utils", "audio_process.py"), "get_embedding",
                             {"np": np, "torch": torch, "rearrange": rearrange})
    get_audio_embedding = compiled(os.path.join(ref_root, "diffsynth", "pipelines", "svi_video_talk.py"), "get_audio_embedding",
                                   {"torch": torch, "audio_prepare_single": lambda path: speech, "get_embedding": get_embedding})
    fake = types.SimpleNamespace(wav2vec_feature_extractor=fe, audio_encoder=model)
    with torch.no_grad():
        iv = torch.from_numpy(np.squeeze(fe(speech, sampling_rate=16000).input_values)).float()
        seq_len = int(len(speech) / 16000 * 25)
        conv = model.feature_extractor(iv[None]).transpose(1, 2)[0]
        interp = tu.linear_interpolation(conv[None], seq_len=seq_len)[0]
        out = model(iv[None], seq_len=seq_len, output_hidden_states=True)
        emb = get_embedding(speech, fe, model)
        starts = [0, 76, seq_len - 20]
        wins = [get_audio_embedding(fake, "unused.wav", 33, audio_start_idx=s) for s in starts]
    hs = torch.stack([h[0] for h in out.hidden_states])
    assert torch.equal(emb, hs[1:].transpose(0, 1))
    np.savez_compressed(os.path.join(HERE, "wav2vec_tiny.npz"), input_values=iv.numpy(), conv_out=conv.numpy(),
                        interp=interp.numpy(), hidden_states=hs.numpy(), last_hidden_state=out.last_hidden_state[0].numpy(),
                        keys=np.array(sorted(model.state_dict().keys())), starts=np.array(starts),
                        windows=np.stack([w.numpy() for w in wins]), num_frames=np.int64(33), seq_len=np.int64(seq_len),
                        seconds=np.float64(6.0), seed=np.int64(0))
    print("audio: conv", tuple(conv.shape), "hidden", tuple(hs.shape), "windows", tuple(wins[0].shape))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    a = ap.parse_args()
    torch.manual_seed(0)
    golden_audio(a.ref)
