"""Inference on the GPU path with the reference's call surface (ZEGGS/generate.py:22-37, 411).

`generate_motion()` is the accelerated core (arrays in, pose tensors out): mel front end -> SpeechEncoder ->
StyleEncoder -> persistent autoregressive decoder, all in libzeggs_b200.so.  `generate_gesture()` keeps the
reference signature; its file-format edges (BVH parse, `preprocess_animation`, BVH write -- SURVEY.md §2 rows 11/13,
out of the accelerated scope) are delegated to the reference's own helpers when they are importable (i.e. when this
runs inside the reference tree as a drop-in), and otherwise pre-processed arrays are accepted / an .npz is written.
"""
import json
import pathlib
import sys
from pathlib import Path
from shutil import copyfile

import numpy as np
import torch

from . import _lib, audio, modules, ops

POSE_KEYS = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]


def load_networks(network_path, device, with_style=True):
    """torch.load of the whole-module pickles (generate.py:130-138); classes named `modules.*` resolve to ours."""
    saved = sys.modules.get("modules")
    sys.modules["modules"] = modules
    try:
        nets = {}
        for n in ("speech_encoder", "decoder") + (("style_encoder",) if with_style else ()):
            nets[n] = torch.load(Path(network_path) / f"{n}.pt", map_location="cpu", weights_only=False).to(device).eval()
    finally:
        if saved is not None:
            sys.modules["modules"] = saved
        else:
            del sys.modules["modules"]
    return nets


def read_wav(path):
    """scipy read + the reference's int->float rescale (audio_files.py:211-236); 16 kHz mono expected (generate.py:161-168).
    16-bit PCM is returned as int16 (the rescale x / 32768 happens on the device), everything else as float32."""
    from scipy.io import wavfile
    return _decode_16k(path, *wavfile.read(str(path)))


def _decode_16k(path, fs, x):
    if x.ndim > 1:
        x = x[:, 0]
    if fs != 16000:
        raise _lib.ZeggsError(f"{path}: expected 16 kHz audio, got {fs} Hz (resample first; the reference shells out to SoX)")
    if x.dtype == np.int16:
        return np.ascontiguousarray(x)             # decoded (x / 32768) by the kernels that consume it
    elif x.dtype == np.int32:
        x = x / 2147483648.0
    elif x.dtype == np.uint8:
        x = ((x / 255.0) - 0.5) * 2
    return x.astype(np.float32)


@torch.no_grad()
def generate_motion(nets, stats, audio_conf, audio_data, style, first_pose, gaze_pos0, dt, temperature=1.0, eps=None,
                    device="cuda"):
    """audio_data [n_samples] (or [N, n_samples]) float32 @16 kHz; style: normalised-able example [T_ex,1134] (raw) or an
    embedding [Z]; first_pose: dict of the 8 first-frame tensors.  Returns the decoder's 8-tuple (batch N)."""
    dev = torch.device(device)
    f = lambda k: torch.as_tensor(stats[k], dtype=torch.float32, device=dev)
    wav = torch.as_tensor(audio_data, dtype=torch.float32, device=dev)
    if wav.dim() == 1:
        wav = wav[None]
    N = wav.shape[0]
    n_frames = int(round(60.0 * (wav.shape[1] / 16000)))                                  # generate.py:170
    feats = audio.preprocess_audio(wav, 60, n_frames, audio_conf, ["mel_spec", "energy"], device=dev)
    if feats.dim() == 2:
        feats = feats[None]
    speech = nets["speech_encoder"]((feats - f("audio_input_mean")) / f("audio_input_std"))
    style = torch.as_tensor(style, dtype=torch.float32, device=dev)
    if style.dim() == 2 and style.shape[-1] == modules.P_IN:                              # a raw example: encode it
        ex = (style[None] - f("anim_input_mean")) / f("anim_input_std")
        z, _, _ = nets["style_encoder"](ex, temperature, eps=eps if eps is not None else None)
    else:
        z = style.reshape(1, -1)
    z = z.expand(N, -1)
    T = speech.shape[1]
    fp = {k: torch.as_tensor(first_pose[k], dtype=torch.float32, device=dev) for k in POSE_KEYS}
    fp = {k: (v[None] if v.dim() == {"root_pos": 1, "root_rot": 1, "root_vel": 1, "root_vrt": 1, "lpos": 2, "ltxy": 3, "lvel": 2, "lvrt": 2}[k] else v)
          for k, v in fp.items()}
    fp = {k: v.expand(N, *v.shape[1:]) for k, v in fp.items()}
    gaze = torch.as_tensor(gaze_pos0, dtype=torch.float32, device=dev).reshape(1, 1, 3).expand(N, T, 3)   # generate.py:374-376
    return nets["decoder"](*[fp[k] for k in POSE_KEYS], gaze, speech, z.unsqueeze(1).repeat(1, T, 1), None,
                           f("anim_input_mean"), f("anim_input_std"), f("anim_output_mean"), f("anim_output_std"), float(dt)), z


def split_by_ratio(length, ratio):
    """Frame ranges of the `stitch` blend (ZEGGS/helpers.py:27-38): consecutive [start, end) with the last one closed at `length`."""
    assert sum(ratio) == 1.0
    end, out = 0.0, []
    for r in ratio:
        s = int(end)
        end = s + r * length
        out.append([s, int(end)])
    out[-1][-1] = length
    return out


def generate_gesture(audio_file, styles, network_path, data_path, results_path, style_encoding_type="example",
                     blend_type="add", blend_ratio=[0.5, 0.5], file_name=None, first_pose=None, temperature=1.0,
                     seed=1234, use_gpu=True, use_script=False):
    """Drop-in for ZEGGS/generate.py:22-411: same arguments, same artefacts (<results_path>/<file_name>.bvh + .wav), same return
    value (the final style encoding: [1,Z] without audio, [1,T,Z] with audio -- generate.py:356-357 re-binds it before returning).
    BVH parsing / feature extraction (zeggs_b200.animation), loudness normalisation + mel (device), the three networks (device),
    the pose -> Euler post-step (device) and the BVH text writer (zeggs_b200.bvhio) are all this package's own."""
    from . import animation, bvhio
    assert (audio_file is None) == (results_path is None)                                # generate.py:84
    if not (use_gpu and torch.cuda.is_available()):
        raise _lib.ZeggsError("zeggs_b200.generate_gesture needs a CUDA device (no CPU fallback)")
    np.random.seed(seed); torch.manual_seed(seed)
    device = torch.device("cuda", torch.cuda.current_device())
    data_path, network_path = Path(data_path), Path(network_path)
    with open(data_path / "data_pipeline_conf.json") as fh:
        conf = json.load(fh)
    with open(data_path / "data_definition.json") as fh:
        details = json.load(fh)
    stats = dict(np.load(data_path / "stats.npz"))
    nets = load_networks(network_path, device, with_style=(style_encoding_type == "example"))
    label_names, dt = details["label_names"], details["dt"]
    f = lambda k: torch.as_tensor(stats[k], dtype=torch.float32, device=device)
    is_path = lambda x: isinstance(x, (pathlib.PurePath, str))

    def features(src, cut=None):
        """path or raw bvh dict (bvh.load layout) -> pose features; the frame range is cut from the RAW animation first (:196-203)."""
        raw = animation.load_bvh(src) if is_path(src) else dict(src)
        if cut is None and is_path(src):
            assert int(np.ceil(1 / raw["frametime"])) == 60                               # generate.py:205-206
        return animation.preprocess_animation(animation.trim(raw, cut))

    if results_path is not None:
        results_path = Path(results_path)
        results_path.mkdir(exist_ok=True)
    encs, last_anim, anim_name = [], None, None
    with torch.no_grad():
        speech = None
        if audio_file is not None:
            from scipy.io import wavfile
            fs, pcm = wavfile.read(str(audio_file))
            if fs == 16000:
                wav = torch.from_numpy(_decode_16k(audio_file, fs, pcm))                 # int16 PCM stays int16: decoded on the device
            else:
                wav = audio.resample(pcm, fs, 16000, device=device)                       # what SoX hands back (audio_files.py:115-146)
            n_frames = int(round(60.0 * (len(wav) / 16000)))                              # generate.py:170
            ac = conf["audio_conf"] if "audio_conf" in conf else conf
            feats = audio.preprocess_audio(wav, 60, n_frames, ac, conf.get("audio_feature_type", ["mel_spec", "energy"]), device=device)
            speech = nets["speech_encoder"]((feats[None] - f("audio_input_mean")) / f("audio_input_std"))
        for style in styles:
            if style_encoding_type == "example":
                if isinstance(style[0], np.ndarray):
                    anim_name = style[1]
                    encs.append(torch.as_tensor(style[0], dtype=torch.float32, device=device)[None])
                else:
                    anim_name = Path(style[0]).stem if is_path(style[0]) else "example"
                    a = features(style[0], style[1]); last_anim = a
                    n = len(a["root_vel"])
                    vec = np.concatenate([a[k].reshape(n, -1) for k in ("root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt")]
                                         + [np.zeros((n, 3), np.float32)], axis=1)        # gaze slot zero (generate.py:240-251)
                    ex = (torch.as_tensor(vec, dtype=torch.float32, device=device) - f("anim_input_mean")) / f("anim_input_std")
                    e, _, _ = nets["style_encoder"](ex[None], temperature)
                    encs.append(e)
            elif style_encoding_type == "label":
                e = torch.zeros((1, len(label_names)), dtype=torch.float32, device=device)
                e[0, label_names.index(style)] = 1.0
                encs.append(e)
                anim_name = style
                assert first_pose is not None                                             # generate.py:270
            else:
                raise ValueError("Unknown style encoding type")
        if blend_type == "stitch":                                                        # generate.py:280-298
            if len(encs) > 1:
                if audio_file is None:
                    final = encs
                else:
                    assert len(styles) == len(blend_ratio)
                    se = split_by_ratio(n_frames, blend_ratio)
                    final = torch.cat([e.unsqueeze(1).repeat((1, se[i][-1] - se[i][0], 1)) for i, e in enumerate(encs)], dim=1)
            else:
                final = encs[0]
        elif blend_type == "add":                                                         # generate.py:299-309
            if len(encs) > 1:
                assert len(encs) == len(blend_ratio)
                final = torch.matmul(torch.stack(encs, dim=1).transpose(2, 1), torch.tensor(blend_ratio, device=device))
            else:
                final = encs[0]
        else:
            raise ValueError(f"unknown blend_type {blend_type!r}")
        if audio_file is None:
            return final
        a = features(first_pose) if first_pose is not None else last_anim                # generate.py:313-354
        if a is None:
            raise _lib.ZeggsError("first_pose is required when no style example provides one (generate.py:313-354)")
        T = speech.shape[1]
        if final.dim() == 2:
            final = final.unsqueeze(1).repeat((1, T, 1))
        g0 = torch.as_tensor(a["gaze_pos"][0], dtype=torch.float32, device=device)
        fp = [torch.as_tensor(a[k][0], dtype=torch.float32, device=device)[None] for k in POSE_KEYS]
        out = nets["decoder"](*fp, g0.reshape(1, 1, 3).repeat(1, T, 1), speech, final, None,
                              f("anim_input_mean"), f("anim_input_std"), f("anim_output_mean"), f("anim_output_std"), float(dt))
        V = dict(zip(POSE_KEYS, out))
        pos, eul = ops.pose_to_bvh_channels(V["root_pos"], V["root_rot"], V["lpos"], V["ltxy"], (0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))
        pos, eul = pos[0].cpu().numpy(), eul[0].cpu().numpy()
    if file_name is None:
        file_name = f"audio_{Path(audio_file).stem}_label_{anim_name}"
    try:
        bvhio.save_bvh(str(results_path / (file_name + ".bvh")), pos, eul, details["parents"], details["bone_names"], "zyx", dt)
        copyfile(audio_file, str(results_path / (file_name + ".wav")))
    except (PermissionError, OSError) as e:                                               # generate.py:407-408
        print(e)
    return final
