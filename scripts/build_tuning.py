"""Build tuning variants of the library for A/B runs on the GPU.
usage: python scripts/build_tuning.py "NCELL=4,JCHUNK=32,TILE_W=16:tag" ..."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magnet_b200 import build
for spec in sys.argv[1:]:
    defs, tag = spec.split(":")
    print(build.build(defines=tuple("MAGNET_" + d for d in defs.split(",")), tag=tag))
