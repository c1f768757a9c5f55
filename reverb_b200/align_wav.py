"""Forced alignment of a known transcript from the command line — the counterpart of the reference's
asr/wenet/bin/alignment.py for one recording of any length, with recognize_wav's flags and output layout
(`<result_dir>/alignment/<audio stem>.ctm`).

    python -m reverb_b200.align_wav --model <dir> --audio_file a.wav --text_file a.txt --result_dir out
"""
from __future__ import annotations

import argparse
import logging
import os
from pathlib import Path


def get_args(argv=None):
    p = argparse.ArgumentParser(description="Align a known transcript to a wav file with the Rev model (CTC forced alignment).")
    p.add_argument("--model", required=True, help="Path to a directory with config and checkpoint, or a pretrained model name")
    p.add_argument("--audio_file", required=True, help="Audio the transcript belongs to (WAV or FLAC natively; other "
                   "containers through torchaudio)")
    src = p.add_mutually_exclusive_group(required=True)
    src.add_argument("--text_file", help="Transcript as text (tokenised with the model's sentencepiece model)")
    src.add_argument("--token_file", help="Transcript as whitespace-separated token ids")
    p.add_argument("--result_dir", required=True, help="The CTM goes to <result_dir>/alignment/<audio stem>.<format>")
    p.add_argument("--gpu", type=int, default=-1, help="gpu id (-1 = current device)")
    p.add_argument("--chunk_size", type=int, default=2051, help="Size of each encoder chunk, in frames")
    p.add_argument("--batch_size", type=int, default=1, help="Number of chunks that are encoded in parallel")
    p.add_argument("--verbatimicity", type=float, default=1.0, help="0.0 = nonverbatim ... 1.0 = verbatim")
    p.add_argument("--blank_penalty", type=float, default=0.0, help="blank penalty")
    p.add_argument("--timings_adjustment", type=float, default=230,
                   help="Subtract timings_adjustment milliseconds from each timestamp")
    p.add_argument("--format", choices=["ctm", "txt"], default="ctm")
    p.add_argument("--log_level", choices=["DEBUG", "INFO", "WARNING", "ERROR", "CRITICAL"], default="INFO")
    return p.parse_args(argv)


def read_transcript(args):
    """-> str (text) or list of token ids."""
    if args.text_file is not None:
        with open(args.text_file, "r", encoding="utf8") as f:
            return " ".join(f.read().split())
    with open(args.token_file, "r", encoding="utf8") as f:
        fields = f.read().split()
    try:
        return [int(x) for x in fields]
    except ValueError as e:
        raise ValueError(f"{args.token_file}: token ids must be integers ({e})") from None


def main(argv=None):
    args = get_args(argv)
    logging.basicConfig(level=args.log_level, format="%(asctime)s %(filename)s %(levelname)s: %(message)s")
    transcript = read_transcript(args)
    if len(transcript) == 0:
        raise ValueError("the transcript is empty, nothing to align")
    from .reverb import load_model
    asr = load_model(args.model, gpu=args.gpu)
    out_dir = os.path.join(args.result_dir, "alignment")
    os.makedirs(out_dir, exist_ok=True)
    target = Path(out_dir) / Path(args.audio_file).with_suffix("." + args.format).name
    text = asr.align(args.audio_file, transcript, format=args.format, verbatimicity=args.verbatimicity,
                     chunk_size=args.chunk_size, batch_size=args.batch_size, blank_penalty=args.blank_penalty,
                     timings_adjustment=args.timings_adjustment)
    with target.open(mode="w") as fp:
        fp.write(text)
    return str(target)


if __name__ == "__main__":
    main()
