#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""Statistics CLI (drop-in for reference wavenet_vocoder/bin/calc_stats.py: same flags, same ``/<type>/mean`` and
``/<type>/scale`` float32 keys).  It runs on the host, as the reference does: scikit-learn's ``StandardScaler.partial_fit``
over the feature files in list order, with the uv column left unnormalised for ``world``.  Feature files may be ``.h5``
or ``.npz`` (``utils.read_hdf5``), and ``world`` / ``mcep`` features made elsewhere are accepted."""
import argparse
import logging

import numpy as np

from pytorchwavenetvocoder_b200.utils import read_hdf5, read_txt, write_hdf5


def calc_stats(file_list, args):
    """CALCULATE STATISTICS (reference calc_stats.py:19-38)."""
    from sklearn.preprocessing import StandardScaler
    scaler = StandardScaler()
    for i, filename in enumerate(file_list):
        logging.info("now processing %s (%d/%d)" % (filename, i + 1, len(file_list)))
        feat = read_hdf5(filename, "/" + args.feature_type)
        scaler.partial_fit(feat)
    mean = scaler.mean_
    scale = scaler.scale_
    if args.feature_type == "world":     # add uv term
        mean[0] = 0.0
        scale[0] = 1.0
    write_hdf5(args.stats, "/" + args.feature_type + "/mean", np.float32(mean))
    write_hdf5(args.stats, "/" + args.feature_type + "/scale", np.float32(scale))


def main(argv=None):
    """RUN CALCULATION OF STATISTICS (reference calc_stats.py:41-86)."""
    parser = argparse.ArgumentParser()
    parser.add_argument("--feats", default=None, required=True, type=str, help="name of the list of hdf5 files")
    parser.add_argument("--stats", default=None, required=True, type=str, help="filename of hdf5 format")
    parser.add_argument("--feature_type", default="world", choices=["world", "melspc", "mcep"], type=str,
                        help="feature type")
    parser.add_argument("--verbose", default=1, type=int, help="log message level")
    args = parser.parse_args(argv)

    fmt = '%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s'
    if args.verbose == 1:
        logging.basicConfig(level=logging.INFO, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    elif args.verbose > 1:
        logging.basicConfig(level=logging.DEBUG, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    else:
        logging.basicConfig(level=logging.WARNING, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
        logging.warning("logging is disabled.")
    for key, value in vars(args).items():
        logging.info("%s = %s" % (key, str(value)))

    file_list = read_txt(args.feats)
    logging.info("number of utterances = %d" % len(file_list))
    calc_stats(file_list, args)


if __name__ == "__main__":
    main()
