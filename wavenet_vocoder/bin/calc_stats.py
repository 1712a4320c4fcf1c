#!/usr/bin/env python
from pytorchwavenetvocoder_b200.bin.calc_stats import *  # noqa
from pytorchwavenetvocoder_b200.bin.calc_stats import main

if __name__ == "__main__":
    main()
