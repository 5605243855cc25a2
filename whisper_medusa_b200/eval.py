"""Evaluation driver: CSV of (audio, sentence[, language]) -> transcripts -> WER / CER -> result CSV.

Mirror of the reference's `whisper_medusa/eval_whisper_medusa.py:21-96` (the caller of the hot path,
SURVEY.md 8(f) rank 1) on top of this package's `WhisperMedusaModel`:

    python -m whisper_medusa_b200.eval --model-name <checkpoint dir> --data-path test.csv \
        --out-file-path out/results.csv [--language en] [--regulation-start 140 --regulation-factor 1.01]

Same arguments, same columns in the result file (`audio,label,prediction,wer,cer,language`), same
scores (`metrics.py` restates jiwer 3.0.3, see there).  Differences, all on the host side:
* audio is read with the standard library (`wave`: PCM 8/16/32-bit, mono or multi-channel -> first
  channel, like `input_speech.squeeze()` on a mono file) or, for other containers, with `torchaudio`
  when its backend is available; resampling to 16 kHz uses `torchaudio.functional.resample`;
* `--frontend engine` (default) feeds the PCM to the engine's own log-mel kernel
  (`generate_from_pcm`); `--frontend hf` computes the features with `WhisperProcessor` on the CPU and
  calls `generate(input_features)` exactly as the reference does (`eval_whisper_medusa.py:46-65`);
* `--chunk-length-s S` (S > 0, at most 30) reads each file at its native rate and transcribes it with
  `model.transcribe(pcm, sampling_rate=sr, chunk_length_s=S)`: recordings of any length, resampled on the GPU
  (the reference accepts at most 30 s).  The default 0 keeps the path above;
* `--no-speech-threshold P --logprob-threshold L`: HF's no-speech rule.  Chunked mode passes both to `transcribe`
  (silent windows add no text); otherwise each clip's `generate` dict output is tested with the same rule
  (`longform.skip_window`) and a silent clip's hypothesis is empty;
* `--temperature 0,0.2,0.4,0.6,0.8,1 --compression-ratio-threshold 2.4 [--logprob-threshold L]`: temperature fallback,
  passed to `transcribe` in chunked mode (refused without `--chunk-length-s`).
"""
from __future__ import annotations

import argparse
import logging
import os
import wave
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from .metrics import compute_cer, compute_wer

SAMPLING_RATE = 16000

__all__ = ["load_audio", "load_audio_native", "evaluate_rows", "evaluate_model", "main"]


def _read_wav(path: str) -> Tuple[np.ndarray, int]:
    with wave.open(path, "rb") as w:
        n_ch, width, sr, n = w.getnchannels(), w.getsampwidth(), w.getframerate(), w.getnframes()
        raw = w.readframes(n)
    if width == 2:
        x = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif width == 4:
        x = np.frombuffer(raw, dtype="<i4").astype(np.float32) / 2147483648.0
    elif width == 1:
        x = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    else:
        raise ValueError(f"{path}: unsupported sample width {width}")
    if n_ch > 1:
        x = x.reshape(-1, n_ch)[:, 0]
    return np.ascontiguousarray(x), sr


def load_audio_native(path: str) -> Tuple[np.ndarray, int]:
    """Mono float32 PCM at the file's own rate, and that rate."""
    try:
        return _read_wav(path)
    except (wave.Error, EOFError):
        import torchaudio   # other containers: whatever backend torchaudio has

        t, sr = torchaudio.load(path)
        return t[0].numpy().astype(np.float32), int(sr)


def load_audio(path: str, sampling_rate: int = SAMPLING_RATE) -> np.ndarray:
    """Mono float32 PCM at `sampling_rate` (reference eval_whisper_medusa.py:42-46)."""
    x, sr = load_audio_native(path)
    if sr != sampling_rate:
        import torch
        import torchaudio.functional as AF

        x = AF.resample(torch.from_numpy(x), sr, sampling_rate).numpy()
    return x


def evaluate_rows(rows: Iterable[Dict], transcribe: Callable[[np.ndarray, str], str], default_language: str = "en",
                  loader: Callable[[str], np.ndarray] = load_audio):
    """Run `transcribe(pcm, language) -> text` over the rows and score the result.

    Returns (wer, cer, table) with `table` the columns of the reference's result file
    (eval_whisper_medusa.py:79-88)."""
    preds: List[str] = []
    gts: List[str] = []
    langs: List[str] = []
    audios: List[str] = []
    for row in rows:
        lang = row.get("language") or default_language
        pcm = loader(row["audio"])
        preds.append(transcribe(pcm, lang))
        sentence = row.get("sentence")
        gts.append("" if sentence is None or (isinstance(sentence, float) and np.isnan(sentence)) else str(sentence))
        langs.append(default_language)     # (the reference records args.language here, eval_whisper_medusa.py:69)
        audios.append(row["audio"])
    wer, wers = compute_wer(preds, gts)
    cer, cers = compute_cer(preds, gts)
    table = {"audio": audios, "label": gts, "prediction": preds, "wer": wers, "cer": cers, "language": langs}
    return wer, cer, table


def evaluate_model(model_name: str, data_path: str, out_file_path: str, language: str = "en",
                   regulation_start: float = 140, regulation_factor: float = 1.0, frontend: str = "engine",
                   device: str = "cuda:0", chunk_length_s: float = 0.0, no_speech_threshold: Optional[float] = None,
                   logprob_threshold: Optional[float] = None, temperature: Optional[Sequence[float]] = None,
                   compression_ratio_threshold: Optional[float] = None):
    import pandas as pd
    import torch
    from transformers import WhisperProcessor

    from . import WhisperMedusaModel
    from .longform import no_speech_rule, skip_window

    if (temperature is not None or compression_ratio_threshold is not None) and chunk_length_s <= 0:
        raise ValueError("--temperature / --compression-ratio-threshold (temperature fallback) need --chunk-length-s")
    fallback = {} if temperature is None else {"temperature": tuple(temperature),
                                               "compression_ratio_threshold": compression_ratio_threshold}
    # (with a schedule, transcribe takes --logprob-threshold alone as a fallback threshold)
    rule = no_speech_rule(no_speech_threshold, None if fallback and no_speech_threshold is None else logprob_threshold)

    data = pd.read_csv(data_path).fillna("")
    processor = WhisperProcessor.from_pretrained(model_name)
    model = WhisperMedusaModel.from_pretrained(model_name).to(device)
    penalty = (regulation_start, regulation_factor) if regulation_factor != 1 else None   # eval_whisper_medusa.py:52-59

    def transcribe(pcm, lang: str) -> str:
        if chunk_length_s > 0:
            x, sr = pcm
            out = model.transcribe(x, sampling_rate=sr, chunk_length_s=chunk_length_s, language=lang,
                                   exponential_decay_length_penalty=penalty, no_speech_threshold=no_speech_threshold,
                                   logprob_threshold=logprob_threshold, **fallback)
            return processor.decode(out[0], skip_special_tokens=True)
        ns = dict(return_dict_in_generate=True, output_no_speech_prob=True) if rule else {}
        if frontend == "hf":
            feats = processor(pcm, return_tensors="pt", sampling_rate=SAMPLING_RATE).input_features
            out = model.generate(feats, language=lang, exponential_decay_length_penalty=penalty, **ns)
        else:
            out = model.generate_from_pcm(pcm, language=lang, exponential_decay_length_penalty=penalty, **ns)
        if rule:
            if skip_window(out.no_speech_prob, out.avg_logprob, no_speech_threshold, logprob_threshold):
                return ""
            out = out.sequences
        return processor.decode(out[0], skip_special_tokens=True)

    with torch.no_grad():
        wer, cer, table = evaluate_rows(data.to_dict("records"), transcribe, default_language=language,
                                        loader=load_audio_native if chunk_length_s > 0 else load_audio)
    logging.info("=======================")
    logging.info(f"WER: {wer}")
    logging.info(f"CER: {cer}")
    logging.info("=======================")
    os.makedirs(os.path.dirname(os.path.abspath(out_file_path)), exist_ok=True)
    pd.DataFrame(table).to_csv(out_file_path, index=False)
    logging.info(f"Results saved to {out_file_path}")
    return wer, cer


def main(argv: Optional[Sequence[str]] = None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model-name", type=str, required=True, help="Path to trained Whisper-Medusa model")
    ap.add_argument("--data-path", type=str, required=True, help="Path to test data csv file (audio, sentence[, language])")
    ap.add_argument("--out-file-path", type=str, required=True, help="Path to output csv file")
    ap.add_argument("--language", type=str, default="en", help="transcribe language")
    ap.add_argument("--regulation-start", type=float, default=140, help="regulation_start for exponential decay")
    ap.add_argument("--regulation-factor", type=float, default=1, help="factor for exponential decay (1 = off)")
    ap.add_argument("--frontend", choices=["engine", "hf"], default="engine", help="log-mel on the GPU (engine) or HF features on the CPU")
    ap.add_argument("--device", type=str, default="cuda:0")
    ap.add_argument("--chunk-length-s", type=float, default=0.0,
                    help="> 0: long-form transcription in windows of this many seconds (at most 30) at the file's own rate")
    ap.add_argument("--no-speech-threshold", type=float, default=None,
                    help="skip a window / clip whose <|nospeech|> probability is above this (needs --logprob-threshold)")
    ap.add_argument("--logprob-threshold", type=float, default=None,
                    help="... and whose average token log-probability is below this")
    ap.add_argument("--temperature", type=str, default=None,
                    help="temperature-fallback schedule, comma-separated, first entry 0 (e.g. 0,0.2,0.4,0.6,0.8,1); "
                         "--chunk-length-s mode")
    ap.add_argument("--compression-ratio-threshold", type=float, default=None,
                    help="decode a window again at the next temperature when its compression ratio is above this")
    args = ap.parse_args(argv)
    logging.basicConfig(format="%(asctime)s - %(name)s - %(levelname)s - %(message)s", level=logging.INFO)
    evaluate_model(args.model_name, args.data_path, args.out_file_path, args.language, args.regulation_start,
                   args.regulation_factor, args.frontend, args.device, args.chunk_length_s, args.no_speech_threshold,
                   args.logprob_threshold,
                   None if args.temperature is None else [float(v) for v in args.temperature.split(",")],
                   args.compression_ratio_threshold)


if __name__ == "__main__":
    main()
