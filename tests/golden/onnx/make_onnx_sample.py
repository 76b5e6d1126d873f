"""Shrinks a real exported ONNX file to tests/golden/onnx/real_export_sample.onnx (< 250 KB) for
tests/test_onnx_import.py::test_reader_parses_a_real_exported_onnx_file.

The source is the libtashkeel model (a torch.onnx export, `deps/libtashkeel/crates/core/data/ort/model.onnx` in the
sonata sources).  Every top-level field of the ModelProto and every graph field except the initialisers is kept byte for
byte; of the initialisers (TensorProto messages, also kept byte for byte) only the smallest ones are kept, up to the
size budget.  Only the length prefixes of the graph and the model change.

    python tests/golden/onnx/make_onnx_sample.py <path to model.onnx>
"""
import os
import sys

BUDGET = 250_000


def varint(b, i):
    v = s = 0
    while True:
        c = b[i]; i += 1
        v |= (c & 0x7F) << s; s += 7
        if c < 0x80:
            return v, i


def enc_varint(v):
    out = bytearray()
    while True:
        c = v & 0x7F; v >>= 7
        out.append(c | (0x80 if v else 0))
        if not v:
            return bytes(out)


def fields(b):
    """(field number, wire type, raw bytes of the whole field, payload) of a serialised message."""
    i = 0
    while i < len(b):
        s = i
        key, i = varint(b, i)
        fno, wt = key >> 3, key & 7
        if wt == 0:
            _, i = varint(b, i); pay = None
        elif wt == 2:
            n, i = varint(b, i); pay = b[i:i + n]; i += n
        elif wt == 5:
            i += 4; pay = None
        elif wt == 1:
            i += 8; pay = None
        else:
            raise ValueError(wt)
        yield fno, wt, b[s:i], pay


def main(src):
    data = open(src, "rb").read()
    out = bytearray()
    for fno, wt, raw, pay in fields(data):
        if fno != 7:
            out += raw
            continue
        other, inits = bytearray(), []
        for gf, gwt, graw, gpay in fields(pay):
            if gf == 5:
                inits.append(graw)
            else:
                other += graw
        kept, size = [], len(out) + len(other)
        for r in sorted(inits, key=len):
            if size + len(r) > BUDGET:
                break
            kept.append(r); size += len(r)
        keep = set(map(bytes, kept))
        graph = bytes(other) + b"".join(r for r in inits if bytes(r) in keep)   # exporter order
        out += enc_varint((7 << 3) | 2) + enc_varint(len(graph)) + graph
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "real_export_sample.onnx")
    open(dst, "wb").write(bytes(out))
    print(dst, len(out))


if __name__ == "__main__":
    main(sys.argv[1])
