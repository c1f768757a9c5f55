"""`reverb` command line — same flags, defaults and output layout as the reference's
asr/wenet/bin/recognize_wav.py (flags :33-145, `<result_dir>/<mode>/<audio stem>.ctm` :177-204).

    python -m reverb_b200.recognize_wav --model <dir> --audio_file a.wav --result_dir out
    python -m reverb_b200.recognize_wav --model <dir> --audio_file calls/*.wav --result_dir out   # batched together
    python -m reverb_b200.recognize_wav --model <dir> --audio_file call.wav --result_dir out --diarization_model dia
        # + out/<mode>/call.stm (a speaker on every word) and out/rttm/call.rttm
"""
from __future__ import annotations

import argparse
import logging
import os
from pathlib import Path

MODES = ["attention", "ctc_greedy_search", "ctc_prefix_beam_search", "attention_rescoring", "joint_decoding"]


def get_args(argv=None):
    from .reverb import get_available_models
    p = argparse.ArgumentParser(description="Run automatic speech recognition on a given wav file using the Rev model.")
    p.add_argument("--audio_file", required=True, nargs="+",
                   help="Audio to transcribe (WAV or FLAC natively; other containers through torchaudio); several "
                        "files are decoded together, in shared batches")
    p.add_argument("--config", default=None, help="Path to config file")
    p.add_argument("--checkpoint", default=None, help="Path to Reverb model checkpoint")
    p.add_argument("--model", default=None,
                   help="Path to directory containing config and checkpoint for a reverb model or the name of a "
                        f"pretrained model from: {','.join(get_available_models())}")
    p.add_argument("--gpu", type=int, default=-1, help="gpu id (this engine always runs on a GPU; -1 = current device)")
    p.add_argument("--tokenizer-symbols", help="Path to tk.units.txt. Overrides the config path.")
    p.add_argument("--bpe-path", help="Path to tk.model. Overrides the config path.")
    p.add_argument("--cmvn-path", help="Path to cmvn. Overrides the config path.")
    p.add_argument("--beam_size", type=int, default=10, help="beam size for search")
    p.add_argument("--length_penalty", type=float, default=0.0,
                   help="length penalty for attention decoding and joint decoding modes")
    p.add_argument("--blank_penalty", type=float, default=0.0, help="blank penalty")
    p.add_argument("--result_dir", required=True, help="asr result file")
    p.add_argument("--batch_size", type=int, default=1, help="Number of chunks that are decoded in parallel")
    p.add_argument("--chunk_size", type=int, default=2051, help="Size of each chunk that is decoded, in frames")
    p.add_argument("--modes", nargs="+", choices=MODES, default=["attention_rescoring"],
                   help="One or more supported decoding mode.")
    p.add_argument("--ctc_weight", type=float, default=0.1, help="ctc weight for attention rescoring decode mode")
    p.add_argument("--decoding_chunk_size", type=int, default=-1,
                   help="decoding chunk size, <0: full chunk (the only mode this engine builds)")
    p.add_argument("--num_decoding_left_chunks", type=int, default=-1, help="number of left chunks for decoding")
    p.add_argument("--simulate_streaming", action="store_true", help="simulate streaming inference")
    p.add_argument("--reverse_weight", type=float, default=0.0,
                   help="right to left weight for attention rescoring decode mode")
    p.add_argument("--overwrite_cmvn", action="store_true",
                   help="overwrite CMVN params in model with those in config file")
    p.add_argument("--verbatimicity", type=float, nargs="+", default=1.0,
                   help="0.0 = nonverbatim ... 1.0 = verbatim; passed to the language-specific layers.  One value, or "
                        "one per --audio_file")
    p.add_argument("--timings_adjustment", type=float, default=230,
                   help="Subtract timings_adjustment milliseconds from each timestamp")
    p.add_argument("--context_list_path", default=None,
                   help="Phrases to boost (names, product terms, jargon), one per line; applies to "
                        "ctc_prefix_beam_search and attention_rescoring")
    p.add_argument("--context_graph_score", type=float, default=6.0,
                   help="Bonus per matched token of a --context_list_path phrase")
    p.add_argument("--diarization_model", default=None,
                   help="Directory with segmentation.pt and embedding.pt (as diarization.infer --pipeline-model): also "
                        "write <result_dir>/<mode>/<stem>.stm and <result_dir>/rttm/<stem>.rttm")
    p.add_argument("--diarization_synthetic", action="store_true",
                   help="Like --diarization_model, with the seeded synthetic diarization weights")
    p.add_argument("--diarization_synthetic_v2", action="store_true",
                   help="Like --diarization_synthetic, with reverb-diarization-v2's (WavLM segmentation)")
    p.add_argument("--log_level", choices=["DEBUG", "INFO", "WARNING", "ERROR", "CRITICAL"], default="INFO")
    args = p.parse_args(argv)
    if isinstance(args.verbatimicity, list):           # one value stays a float; else one per --audio_file
        if len(args.verbatimicity) not in (1, len(args.audio_file)):
            p.error(f"--verbatimicity takes one value or one per --audio_file ({len(args.audio_file)}), "
                    f"got {len(args.verbatimicity)}")
        if len(args.verbatimicity) == 1:
            args.verbatimicity = args.verbatimicity[0]
    return args


def output_names(audio_files) -> list:
    """`<stem>.ctm` of every input; two inputs with the same stem would write the same file."""
    names = [Path(f).with_suffix(".ctm").name for f in audio_files]
    seen = {}
    for f, n in zip(audio_files, names):
        if n in seen:
            raise ValueError(f"--audio_file {seen[n]} and {f} would both write {n}")
        seen[n] = f
    return names


def main(argv=None):
    args = get_args(argv)
    names = output_names(args.audio_file)
    logging.basicConfig(level=args.log_level, format="%(asctime)s %(filename)s %(levelname)s: %(message)s")
    from .reverb import ReverbASR, load_model
    by_name = args.model is not None
    by_files = args.checkpoint is not None and args.config is not None
    if by_name == by_files:
        raise RuntimeError("One of either --model or (--checkpoint and --config) must be set.")
    if by_name:
        asr = load_model(args.model, gpu=args.gpu)
    else:
        asr = ReverbASR(args.config, args.checkpoint, cmvn_path=args.cmvn_path,
                        tokenizer_symbols=args.tokenizer_symbols, bpe_path=args.bpe_path, gpu=args.gpu,
                        overwrite_cmvn=args.overwrite_cmvn)
    out_dirs = []
    for mode in args.modes:
        out_dirs.append(Path(args.result_dir) / mode)
        os.makedirs(out_dirs[-1], exist_ok=True)
    diarization = None
    if args.diarization_model or args.diarization_synthetic or args.diarization_synthetic_v2:
        from .diarization.infer import load_pipeline
        diarization = load_pipeline(args.diarization_model,
                                    synthetic="v2" if args.diarization_synthetic_v2 else args.diarization_synthetic)
        os.makedirs(Path(args.result_dir) / "rttm", exist_ok=True)
    graph = asr.context_graph(args.context_list_path, args.context_graph_score) if args.context_list_path else None
    results = asr.transcribe_files(
        args.audio_file, modes=args.modes, format="ctm", verbatimicity=args.verbatimicity,
        chunk_size=args.chunk_size, batch_size=args.batch_size, beam_size=args.beam_size,
        decoding_chunk_size=args.decoding_chunk_size, num_decoding_left_chunks=args.num_decoding_left_chunks,
        ctc_weight=args.ctc_weight, simulate_streaming=args.simulate_streaming, reverse_weight=args.reverse_weight,
        blank_penalty=args.blank_penalty, length_penalty=args.length_penalty,
        timings_adjustment=args.timings_adjustment, context_graph=graph)
    for name, (path, outputs) in zip(names, results):
        for out_dir, text in zip(out_dirs, outputs):
            with (out_dir / name).open(mode="w") as fp:
                fp.write(text)
        if diarization is not None:
            from .reverb import speaker_outputs
            rttm, stms = speaker_outputs(diarization, path, outputs)
            stem = Path(name).stem
            with (Path(args.result_dir) / "rttm" / f"{stem}.rttm").open(mode="w") as fp:
                fp.write(rttm)
            for out_dir, text in zip(out_dirs, stms):
                with (out_dir / f"{stem}.stm").open(mode="w") as fp:
                    fp.write(text)


if __name__ == "__main__":
    main()
