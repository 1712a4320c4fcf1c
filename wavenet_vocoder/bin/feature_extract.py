#!/usr/bin/env python
from pytorchwavenetvocoder_b200.bin.feature_extract import *  # noqa
from pytorchwavenetvocoder_b200.bin.feature_extract import main

if __name__ == "__main__":
    main()
