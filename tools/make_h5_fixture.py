"""Write tests/golden/whenet_h5_shrunk.h5.gz: the reference's WHENet.h5 with every metadata byte kept and the data
of large tensors thinned out, small enough to live in the repository.

  python tools/make_h5_fixture.py path/to/WHENet.h5

Every byte outside the datasets' data ranges (superblock, object headers, local and global heaps, B-trees, attributes)
is copied unchanged, so the file has the original's exact layout.  Tensors of at most FULL elements keep all their
data; larger ones keep their first and last EDGE elements and are zero in between.  tests/test_weights_reader.py reads
it with h5lite and compares the kept elements with the committed npz.
"""
import gzip
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FULL = 512
EDGE = 128
OUT = os.path.join(ROOT, "tests", "golden", "whenet_h5_shrunk.h5.gz")


def main(src):
    from whenet_b200 import h5lite
    f = h5lite.H5File(src)
    buf = bytearray(f.buf)
    for _path, addr in f.visit():
        daddr, dsize = struct.unpack_from("<QQ", f.obj(addr).first(0x08), 2)
        n = dsize // 4                                   # every dataset of WHENet.h5 is float32
        if n > FULL:
            buf[daddr + EDGE * 4:daddr + dsize - EDGE * 4] = bytes(dsize - 2 * EDGE * 4)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as g:
        g.write(bytes(buf))
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main(sys.argv[1])
