"""python -m tactics2d_b200.map osm_root  - compile the OSM maps below osm_root (the reference's ``data`` directory) into
segment tiles."""
import sys

from . import compile_tiles, load_collidable_segments

if len(sys.argv) != 2:
    sys.exit("usage: python -m tactics2d_b200.map <osm_root>")
root = sys.argv[1]
for name in compile_tiles(root):
    seg, b = load_collidable_segments(name)
    print(f"{name}: {len(seg)} collidable segments, bounds {b}")
