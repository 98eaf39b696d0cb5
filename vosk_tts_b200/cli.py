"""`vosk-tts` command line (flags of vosk_tts/cli.py:12-43) on top of the CUDA engine."""
import argparse
import json
import logging
import sys

from .model import Model, list_languages, list_models
from .synth import Synth


def main(argv=None):
    p = argparse.ArgumentParser(description="Synthesize input")
    p.add_argument("--model", "-m", type=str, help="model path")
    p.add_argument("--list-models", default=False, action="store_true", help="list available models")
    p.add_argument("--list-languages", default=False, action="store_true", help="list available languages")
    p.add_argument("--model-name", "-n", type=str, help="select model by name")
    p.add_argument("--lang", "-l", default="en-us", type=str, help="select model by language")
    p.add_argument("--input", "-i", type=str, help="input string")
    p.add_argument("--speaker", "-s", type=int, help="speaker id for multispeaker model")
    p.add_argument("--speech-rate", "-r", type=float, default=1.0, help="speech rate of the synthesis")
    p.add_argument("--output", "-o", default="out.wav", type=str, help="optional output filename path")
    p.add_argument("--log-level", default="INFO", help="logging level")
    p.add_argument("--device", type=int, default=0, help="CUDA device index (extension)")
    p.add_argument("--precision", type=int, default=1, choices=(0, 1, 2, 3),
                   help="engine precision mode (extension).  VITS voices: 0 fp32 FFMA, 1 flow and decoder on the tensor cores, "
                        "2 the text encoder as well, 3 as 2 with exact durations.  Multistream voices: 0 fp32 FFMA, 1 vocoder and "
                        "BERT on the tensor cores, 2 the flow-matching decoder as well, 3 as 1")
    p.add_argument("--convert-from", type=str, help="voice conversion (extension): re-voice this mono WAV as --speaker")
    p.add_argument("--source-speaker", type=int, help="speaker id of the --convert-from recording")
    p.add_argument("--align", type=str, metavar="WAV",
                   help="forced alignment (extension): print the phoneme segments of --input in this mono WAV as JSON")
    p.add_argument("--resample", default=False, action="store_true",
                   help="--convert-from / --align: read a 16-bit WAV at any rate, mono or stereo, and resample it on the GPU")
    args = p.parse_args(argv)
    logging.getLogger().setLevel(args.log_level.upper())
    if args.list_models:
        list_models()
        return 0
    if args.list_languages:
        list_languages()
        return 0
    if args.convert_from:
        if args.source_speaker is None or args.speaker is None:
            p.error("--convert-from needs --source-speaker and --speaker (the target)")
        model = Model(args.model, args.model_name, args.lang, device=args.device, voice_conversion=True)
        extra = {"resample": True} if args.resample else {}
        Synth(model).convert(args.convert_from, args.output, args.source_speaker, args.speaker, **extra)
        return 0
    if args.align:
        if not args.input:
            p.error("--align needs --input (the transcript of the recording)")
        model = Model(args.model, args.model_name, args.lang, device=args.device, voice_conversion=True)
        extra = {"resample": True} if args.resample else {}
        print(json.dumps(Synth(model).align(args.align, args.input, speaker_id=args.speaker, **extra)))
        return 0
    if not args.input:
        logging.info("Please specify input text or file")
        return 1
    model = Model(args.model, args.model_name, args.lang, device=args.device, precision=args.precision)
    Synth(model).synth(args.input, args.output, speaker_id=args.speaker, speech_rate=args.speech_rate)
    return 0


if __name__ == "__main__":
    sys.exit(main())
