"""Command line front-end, flag-compatible with the reference's
``scripts/ina_speech_segmenter.py`` (:45-84): -i/-o/-s/-d/-g/-b/-e/-r, plus
``--devices`` to spread the input files over several local GPUs (file-level
parallelism, what the reference's Pyro4 farm did across hosts)."""
import argparse
import glob
import os
import sys
import warnings

description = """Do Speech/Music(/Noise) and Male/Female segmentation and store segmentations into CSV files. Segments labelled 'noEnergy' are discarded from music, noise, speech and gender analysis. 'speech', 'male' and 'female' labels include speech over music and speech over noise. 'music' and 'noise' labels are pure segments that are not supposed to contain speech.
"""


def _strtobool(v):
    v = v.lower()
    if v in ('y', 'yes', 't', 'true', 'on', '1'):
        return True
    if v in ('n', 'no', 'f', 'false', 'off', '0'):
        return False
    raise ValueError('invalid truth value %r' % v)


def build_parser():
    p = argparse.ArgumentParser(description=description)
    p.add_argument('-i', '--input', nargs='+', required=True, help='Input media to analyse (paths, glob patterns or http urls)')
    p.add_argument('-o', '--output_directory', required=True, help='Directory used to store segmentations')
    p.add_argument('-s', '--batch_size', type=int, default=32, help='kept for compatibility (the GPU kernels batch internally)')
    p.add_argument('-d', '--vad_engine', choices=['sm', 'smn'], default='smn')
    p.add_argument('-g', '--detect_gender', choices=['true', 'false'], default='True')
    p.add_argument('-b', '--ffmpeg_binary', default='ffmpeg', help='ffmpeg binary; "None" disables ffmpeg (WAV input only)')
    p.add_argument('-e', '--export_format', choices=['csv', 'textgrid'], default='csv')
    p.add_argument('-r', '--energy_ratio', default=0.03, type=float)
    p.add_argument('--devices', default='0', help='comma-separated CUDA ordinals; files are dealt round-robin, one process per GPU')
    return p


def _worker(device, files, outs, args, detect_gender, ffmpeg):
    from . import Segmenter
    seg = Segmenter(vad_engine=args.vad_engine, detect_gender=detect_gender, ffmpeg=ffmpeg,
                    energy_ratio=args.energy_ratio, batch_size=args.batch_size, device=device)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return seg.batch_process(files, outs, verbose=True, output_format=args.export_format)


def main(argv=None):
    args = build_parser().parse_args(argv)
    ffmpeg = args.ffmpeg_binary
    if ffmpeg.lower() == 'none' or ffmpeg == '':
        print('Disabling ffmpeg. WAV input only.')
        ffmpeg = None
    input_files = []
    for e in args.input:
        input_files += [e] if e.startswith('http') else glob.glob(e)
    assert len(input_files) > 0, 'No existing media selected for analysis! Bad values provided to -i (%s)' % args.input
    odir = args.output_directory.strip(' \t\n\r').rstrip('/')
    assert os.access(odir, os.W_OK), 'Directory %s is not writable!' % odir
    detect_gender = _strtobool(args.detect_gender)
    base = [os.path.splitext(os.path.basename(e))[0] for e in input_files]
    output_files = [os.path.join(odir, e + '.' + args.export_format) for e in base]
    devices = [int(d) for d in args.devices.split(',') if d != '']
    if len(devices) <= 1:
        return _worker(devices[0] if devices else 0, input_files, output_files, args, detect_gender, ffmpeg)
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    procs = []
    for k, dev in enumerate(devices):
        p = ctx.Process(target=_worker, args=(dev, input_files[k::len(devices)], output_files[k::len(devices)], args, detect_gender, ffmpeg))
        p.start()
        procs.append(p)
    for p in procs:
        p.join()
    failed = [(dev, p.exitcode) for dev, p in zip(devices, procs) if p.exitcode != 0]
    if failed:                                   # a crashed worker must not look like success to the caller's shell
        sys.exit('worker(s) failed (device, exit code): %r' % failed)
    return None


if __name__ == '__main__':
    main()
