"""scripts/preprocess/compress_metadata.py: a phrase dump's metadata -> meta_compressed.pkl (artifacts.write_meta), which MIPS keeps in
memory with a PQ index.  Same flags and defaults as the reference script.

    python -m densephrases_b200.compress_metadata --input_dump_dir DUMP/phrase --output_dir DUMP"""
import argparse

from . import artifacts


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('--input_dump_dir', type=str, default='dump/sbcd_sqdqgnqqg_inb64_s384_sqdnq_pinb2_0_20181220_concat/dump/phrase')
    parser.add_argument('--output_dir', type=str, default='./')
    args = parser.parse_args(argv)
    print(artifacts.write_meta(args.input_dump_dir, args.output_dir))


if __name__ == '__main__':
    main()
