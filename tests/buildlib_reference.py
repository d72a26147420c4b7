"""Plain restatement of `megahit_core buildlib` (sequence_lib.cpp, fastx_reader.cpp, paired_fastx_reader.cpp, kseq.h,
sequence_package.h): FASTA/FASTQ text in, the `.bin` image and `.lib_info` text out.  Byte-level and unoptimised on
purpose; it is what the GPU path is checked against.

Rules restated:
- kseq: a record starts at the next '>' or '@' anywhere (after a FASTQ record, or at the start of a file) or at the
  line that ended the previous FASTA record; the header is the rest of that line (a bare marker as the unterminated
  last line is end of file); sequence lines run until a line starting with '>', '+' or '@' (empty lines skipped);
  a '+' line opens the quality block, read line by line until it is at least as long as the sequence.  A trailing
  '\\r' is dropped from the accumulated string when it is longer than one byte (not for a one-byte sequence line
  without a final newline).  A quality block of another length, or a '+' line that ends the file, is an error.
- FastxReader::Read / PairedFastxReader::Read batches (4 Mi reads or 2^28 bases): an error ends the current batch;
  an error (or end of file) at the start of a batch ends the library.
- TrimN keeps the first maximal N-free run; an empty read becomes the one-base read "A"; 2-bit packing, first base
  in the most significant bits, A/C/G/T (either case) -> 0..3, every other byte -> 0.
"""
import struct

BATCH_READS = 1 << 22
BATCH_BASES = 1 << 28
ERR = None


def kseq_records(data: bytes):
    """Every kseq_read result of one stream in order: the raw sequence (bytes) or ERR; ends at end of file."""
    n = len(data)
    pos = 0
    last_char = False  # the marker of the next header has been consumed
    out = []
    while True:
        if not last_char:
            while pos < n and data[pos] not in (0x3E, 0x40):
                pos += 1
            if pos >= n:
                return out
            pos += 1
        # header: the rest of the line; a bare marker at the end of the data is end of file
        if pos >= n:
            return out
        nl = data.find(b"\n", pos)
        pos = n if nl < 0 else nl + 1
        seq = bytearray()
        c = -1
        while pos < n:
            c = data[pos]
            pos += 1
            if c in (0x3E, 0x2B, 0x40):
                break
            if c == 0x0A:
                c = -1
                continue
            seq.append(c)
            nl = data.find(b"\n", pos)
            tail_end = n if nl < 0 else nl
            got = tail_end > pos or nl >= 0
            seq += data[pos:tail_end]
            pos = tail_end + 1 if nl >= 0 else n
            if got and len(seq) > 1 and seq[-1] == 0x0D:
                del seq[-1]
            c = -1
        if c in (0x3E, 0x40):
            last_char = True
        if c != 0x2B:
            out.append(bytes(seq))
            if c == -1:
                return out
            continue
        # '+' line
        nl = data.find(b"\n", pos)
        if nl < 0:
            out.append(ERR)
            return out
        pos = nl + 1
        qual = 0
        while True:
            if pos >= n:
                break
            nl = data.find(b"\n", pos)
            tail_end = n if nl < 0 else nl
            qual += tail_end - pos
            if qual > 1 and data[tail_end - 1] == 0x0D and tail_end > pos:
                qual -= 1
            pos = tail_end + 1 if nl >= 0 else n
            if qual >= len(seq):
                break
        last_char = False
        out.append(bytes(seq) if qual == len(seq) else ERR)


def trim_n(s: bytes) -> bytes:
    b = 0
    while b < len(s) and s[b] in b"Nn":
        b += 1
    e = b
    while e < len(s) and s[e] not in b"Nn":
        e += 1
    return s[b:e]


_CODE = bytearray(256)
for _c, _v in zip(b"ACGTacgt", (0, 1, 2, 3, 0, 1, 2, 3)):
    _CODE[_c] = _v


def pack_read(s: bytes) -> bytes:
    if len(s) == 0:
        s = b"A"
    words = [0] * ((len(s) + 15) // 16)
    for i, c in enumerate(s):
        words[i // 16] |= _CODE[c] << (30 - 2 * (i % 16))
    return struct.pack(f"<I{len(words)}I", len(s), *words)


def library_reads(streams, paired: bool):
    """The trimmed reads one library contributes: streams = record lists from kseq_records (one, or two for pe)."""
    reads = []
    i_batch = bases = 0
    if not paired:
        for rec in streams[0]:
            if rec is ERR:
                if i_batch == 0:
                    return reads
                i_batch = bases = 0
                continue
            t = trim_n(rec)
            reads.append(t)
            bases += len(t)
            i = i_batch
            i_batch += 1
            if (bases >= BATCH_BASES and i % 2 == 1) or i_batch == BATCH_READS:
                i_batch = bases = 0
        return reads
    a, b = streams
    for j in range(min(len(a), len(b))):
        if a[j] is ERR or b[j] is ERR:
            if i_batch == 0:
                return reads
            i_batch = bases = 0
            continue
        ta, tb = trim_n(a[j]), trim_n(b[j])
        reads += [ta, tb]
        bases += len(ta) + len(tb)
        i_batch += 2
        if bases >= BATCH_BASES or i_batch >= BATCH_READS:
            i_batch = bases = 0
    return reads


class LibError(Exception):
    pass


def parse_lib_file(text: str):
    """(metadata, type, [files]) per block, with the reference's istream semantics (getline, >>, getline)."""
    import io
    s = io.StringIO(text)
    blocks = []
    typ, f1, f2 = "", "", ""

    def word():
        c = s.read(1)
        while c and c.isspace():
            c = s.read(1)
        if not c:
            return None
        w = []
        while c and not c.isspace():
            w.append(c)
            c = s.read(1)
        if c:
            s.seek(s.tell() - 1)
        return "".join(w)

    while True:
        line = s.readline()
        if line == "":
            break
        meta = line[:-1] if line.endswith("\n") else line
        t = word()
        ok = t is not None
        if ok:
            typ = t
        if typ == "pe":
            w = word() if ok else None
            ok = ok and w is not None
            if ok:
                f1 = w
            w = word() if ok else None
            ok = ok and w is not None
            if ok:
                f2 = w
            blocks.append((meta, typ, [f1, f2]))
        elif typ in ("se", "interleaved"):
            w = word() if ok else None
            ok = ok and w is not None
            if ok:
                f1 = w
            blocks.append((meta, typ, [f1]))
        else:
            raise LibError("Valid types: pe, se, interleaved")
        if not ok:  # the stream has failed: the next getline ends the loop
            break
        s.readline()
    return blocks


def buildlib(libs):
    """libs = [(metadata, type, [file bytes])] -> (bin bytes, lib_info text).  Raises LibError as the reference exits."""
    out = bytearray()
    total_reads = total_bases = 0
    info = []
    for meta, typ, datas in libs:
        recs = [kseq_records(d) for d in datas]
        reads = library_reads(recs, typ == "pe")
        if typ != "se" and len(reads) % 2:
            raise LibError(f"PE library number of reads is odd: {len(reads)}!")
        begin = total_reads
        max_len = 0
        for r in reads:
            out += pack_read(r)
            L = max(len(r), 1)
            total_bases += L
            max_len = max(max_len, L)
        total_reads += len(reads)
        info.append(f"{meta}\n{begin} {total_reads} {max_len} {0 if typ == 'se' else 1}\n")
    return bytes(out), f"{total_bases} {total_reads}\n" + "".join(info)
