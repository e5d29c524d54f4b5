"""Junction-jump test data and a plain-Python restatement of mm_jump_split's decisions (jump.c:7-194).

make_data() builds, from one seed: a small genome of spliced genes (GT..AG introns), spliced reads whose first or last exon overhangs
by 1 to 30 bases (with a mismatch or an N in some overhangs, on both strands), an annotation BED (BED12 transcripts, duplicated
introns, opposite-strand copies of the same intron, decoy junctions a few bases off the true sites) and, per read, the hit an aligner
that stopped short of the overhangs would report. decide() is what K5 computes for one hit."""
import bisect
import os
import numpy as np

NT = b"ACGT"
COMP = bytes.maketrans(b"ACGTN", b"TGCAN")
NT4 = np.full(256, 4, dtype=np.uint8)
for _i, _c in enumerate(b"ACGT"):
    NT4[_c] = NT4[_c + 32] = _i
NT4[ord("U")] = NT4[ord("u")] = 3
MM_JUNC_ANNO = 1


def revcomp(s):
    return s.translate(COMP)[::-1]


def _rand_seq(rng, n):
    return bytes(NT[i] for i in rng.integers(0, 4, n))


def make_data(seed=11, n_contigs=2, genes_per_contig=6, reads_per_gene=40, n_exons=(3, 6)):
    rng = np.random.default_rng(seed)
    contigs, genes = [], []
    for c in range(n_contigs):
        seq = bytearray(_rand_seq(rng, 400))
        for g in range(genes_per_contig):
            exons = []
            for e in range(int(rng.integers(*n_exons))):
                if e:
                    intron = bytearray(_rand_seq(rng, int(rng.integers(120, 900))))
                    intron[:2], intron[-2:] = b"GT", b"AG"
                    seq += intron
                st = len(seq)
                seq += _rand_seq(rng, int(rng.integers(60, 200)))
                exons.append((st, len(seq)))
            genes.append((c, exons, "+" if rng.random() < 0.7 else "-"))
            seq += _rand_seq(rng, int(rng.integers(200, 600)))
        contigs.append(bytes(seq))
    names = ["chr%d" % (c + 1) for c in range(n_contigs)]
    bed = []
    for gi, (c, ex, strand) in enumerate(genes):
        sizes = ",".join(str(e - s) for s, e in ex)
        starts = ",".join(str(s - ex[0][0]) for s, e in ex)
        bed.append("%s\t%d\t%d\ttx%d\t0\t%s\t%d\t%d\t0\t%d\t%s,\t%s," % (names[c], ex[0][0], ex[-1][1], gi, strand, ex[0][0], ex[-1][1], len(ex), sizes, starts))
        for k in range(1, len(ex)):
            st, en = ex[k - 1][1], ex[k][0]
            if rng.random() < 0.3:  # the same intron again, same strand or the opposite one (the merged entry keeps one strand)
                bed.append("%s\t%d\t%d\tdup\t0\t%s" % (names[c], st, en, strand if rng.random() < 0.5 else "+-"[strand == "+"]))
            if rng.random() < 0.4:  # decoys a few bases off the true sites
                d1, d2 = int(rng.integers(-4, 5)), int(rng.integers(-4, 5))
                if d1 or d2:
                    bed.append("%s\t%d\t%d\tdecoy\t0\t%s" % (names[c], st + d1, en + d2, strand))
            if rng.random() < 0.15:  # a second junction from the same donor: two candidates can match one end
                bed.append("%s\t%d\t%d\talt\t0\t%s" % (names[c], st, en + int(rng.integers(-3, 4)) * 3, strand))
    reads, hits = [], []
    for gi, (c, ex, strand) in enumerate(genes):
        g = contigs[c]
        for r in range(reads_per_gene):
            k0 = int(rng.integers(0, len(ex) - 1))
            k1 = int(rng.integers(k0 + 1, len(ex)))
            ov_l = [1, 2, 3, 4, 5, 8, 12, 20, 30][int(rng.integers(0, 9))] if rng.random() < 0.8 else 0
            ov_r = [1, 2, 3, 4, 5, 8, 12, 20, 30][int(rng.integers(0, 9))] if rng.random() < 0.8 else 0
            ov_l = min(ov_l, ex[k0][1] - ex[k0][0] - 1)
            ov_r = min(ov_r, ex[k1][1] - ex[k1][0] - 1)
            inner = ex[k0 + 1:k1] if k1 > k0 + 1 else []
            if ov_l == 0 and ov_r == 0:
                continue
            if not inner:  # the aligned part must be long enough (more than ext + 20 bases on each end): take whole exons
                inner, ov_r = ex[k0 + 1:k1 + 1], 0
                if k1 + 1 < len(ex) and rng.random() < 0.5:
                    ov_r = min(int(rng.integers(1, 31)), ex[k1 + 1][1] - ex[k1 + 1][0] - 1)
                    k1 += 1
                else:
                    k1 = k0 + len(inner) + 1
            segs = []
            if ov_l:
                segs.append(bytearray(g[ex[k0][1] - ov_l:ex[k0][1]]))
            for s, e in inner:
                segs.append(bytearray(g[s:e]))
            if ov_r and k1 < len(ex):
                segs.append(bytearray(g[ex[k1][0]:ex[k1][0] + ov_r]))
            else:
                ov_r = 0
            u = rng.random()
            for ov, si in ((ov_l, 0), (ov_r, len(segs) - 1)):
                if ov and u < 0.12:
                    p = int(rng.integers(0, ov))
                    segs[si][p] = NT[(NT.index(segs[si][p]) + 1) % 4]
                elif ov and u < 0.2:
                    segs[si][int(rng.integers(0, ov))] = ord("N")
            t = b"".join(bytes(s) for s in segs)
            a0, a1 = ov_l, len(t) - ov_r  # the aligned part of t
            rs, re = inner[0][0], inner[-1][1]
            cig = []
            for j, (s, e) in enumerate(inner):
                if j:
                    cig.append((s - inner[j - 1][1]) << 4 | 3)
                cig.append((e - s) << 4)
            if rng.random() < 0.25 and len(inner) > 1:  # an end that stops inside an exon: single-M CIGAR when one exon is left
                inner1 = inner[:1]
                re, a1 = inner1[0][1], ov_l + inner1[0][1] - inner1[0][0]
                cig = [(re - rs) << 4]
                t = t[:a1] if rng.random() < 0.5 else t
            rev = int(rng.random() < 0.5)
            q = revcomp(t) if rev else t
            qs, qe = (len(t) - a1, len(t) - a0) if rev else (a0, a1)
            reads.append(("r%d_%d" % (gi, r), q))
            hits.append(dict(read=len(reads) - 1, rid=c, rs=rs, re=re, qs=qs, qe=qe, rev=rev, cigar=cig))
    return dict(contigs=contigs, names=names, bed=bed, reads=reads, hits=hits)


def write_data(d, dirname):
    os.makedirs(dirname, exist_ok=True)
    with open(os.path.join(dirname, "ref.fa"), "w") as f:
        for n, s in zip(d["names"], d["contigs"]):
            f.write(">%s\n%s\n" % (n, s.decode()))
    with open(os.path.join(dirname, "reads.fa"), "w") as f:
        for n, s in d["reads"]:
            f.write(">%s\n%s\n" % (n, s.decode()))
    with open(os.path.join(dirname, "anno.bed"), "w") as f:
        f.write("\n".join(d["bed"]) + "\n")
    return dirname


def hit_variants(data, rng):
    """the generator's hits, and copies moved by a few bases / with a clipped CIGAR end, so that decoys and trims are exercised"""
    out = list(data["hits"])
    for h in data["hits"]:
        for _ in range(3):
            x = dict(h)
            d1, d2 = int(rng.integers(-6, 7)), int(rng.integers(-6, 7))
            cig = list(h["cigar"])
            if cig[0] >> 4 <= 40 or cig[-1] >> 4 <= 40 or (len(cig) == 1 and (cig[0] >> 4) - abs(d1) - abs(d2) <= 40):
                continue
            if h["rev"]:
                x["qe"], x["qs"] = h["qe"] - d1, h["qs"] + d2
            else:
                x["qs"], x["qe"] = h["qs"] + d1, h["qe"] - d2
            x["rs"], x["re"] = h["rs"] + d1, h["re"] - d2
            if len(cig) == 1:
                cig[0] -= (d1 + d2) << 4
            else:
                cig[0] -= d1 << 4
                cig[-1] -= d2 << 4
            x["cigar"] = cig
            if 0 <= x["qs"] < x["qe"] <= len(data["reads"][h["read"]][1]):
                out.append(x)
    return out


# ---- the restatement ----
def jump_get(table, seq_len, st, en):
    """mm_idx_jump_get (index.c:932-959): entries with off in (st, en], en clamped to the contig length. table: sorted entries of one
    contig as (off, off2, flag) tuples."""
    if en < 0 or en > seq_len:
        en = seq_len
    offs = [e[0] for e in table]
    lo, hi = bisect.bisect_right(offs, st), bisect.bisect_right(offs, en)
    return table[lo:hi] if hi > lo else []


def _check(st, rev, qlen, seq_len, ext, is_left):
    rs, re, qs, qe, n_cigar, first, last = st
    if n_cigar <= 0:
        return False
    e = int(not rev) ^ int(not is_left)
    clip = qs if e == 0 else qlen - qe
    c = first if is_left else last
    clen = c >> 4 if c & 0xf == 0 else 0
    if clen <= ext:
        return False
    return clip < rs if is_left else clip < seq_len - re


def _side(st, rev, q4, tseq, seq_len, table, a, b, jmm, is_left):
    rs, re, qs, qe = st[:4]
    qlen = len(q4)
    ext = 1 + (b + a - 1) // a + 1
    none = (0, 0, 0, 0, 0)
    if not _check(st, rev, qlen, seq_len, ext + 20, is_left):
        return none
    clip = (qs if not rev else qlen - qe) if is_left else (qlen - qe if not rev else qs)
    extt, L = min(clip, ext), clip + ext
    cand = jump_get(table, seq_len, rs - extt, rs + ext) if is_left else jump_get(table, seq_len, re - ext, re + extt)
    if is_left:
        qq = q4[:L] if not rev else np.where(q4[::-1][:L] >= 4, q4[::-1][:L], 3 - q4[::-1][:L])
    else:
        qq = q4[qlen - L:] if not rev else np.where(q4[L - 1::-1] >= 4, q4[L - 1::-1], 3 - q4[L - 1::-1])
    best = {True: [-1, 0, 0], False: [-1, 0, 0]}  # anno: i0, n, mm0
    for i, (off, off2, flag) in enumerate(cand):
        if is_left:
            if off2 >= off or off - off2 < 6 or off2 < L:
                continue
            tl1 = clip + (off - rs)
            t = np.concatenate([tseq[off2 - tl1:off2], tseq[off:rs + ext]])
            mis = (qq != t) | (qq > 3) | (t > 3)
            mm1, mm2 = int(mis[:tl1].sum()), int(mis[tl1:].sum())
        else:
            if off2 <= off or off2 - off < 6 or off2 + L > seq_len:
                continue
            tl1 = clip + (re - off)
            t = np.concatenate([tseq[re - ext:off], tseq[off2:off2 + tl1]])
            mis = (qq != t) | (qq > 3) | (t > 3)
            mm2, mm1 = int(mis[:L - tl1].sum()), int(mis[L - tl1:].sum())
        if mm1 == 0 and mm2 <= 1:
            x = best[bool(flag & MM_JUNC_ANNO)]
            if is_left or x[0] < 0:
                x[0], x[2] = i, mm1 + mm2
            x[1] += 1
    x = best[True] if best[True][1] > 0 else best[False]
    m, i0, mm0 = x[1], x[0], x[2]
    if m == 0:
        return none
    off, off2 = cand[i0][0], cand[i0][1]
    l = off - rs if is_left else re - off
    if m == 1 and clip + l >= jmm:
        act = 2
    elif (off > rs) if is_left else (re > off):
        act = 1
    else:
        act = 0
    return (act, l, off, off2, mm0)


def decide(hit, q, tseq, table, a, b, jump_min_match):
    """((act, l, off, off2, mm0) of the left end, then of the right end) for one hit; q: the read (ASCII bytes); tseq: the contig as
    nt4 (numpy uint8); table: the contig's jump entries (off, off2, flag)"""
    q4 = NT4[np.frombuffer(q, dtype=np.uint8)]
    cig = hit["cigar"]
    st = [hit["rs"], hit["re"], hit["qs"], hit["qe"], len(cig), cig[0], cig[-1]]
    rev, qlen, seq_len = hit["rev"], len(q), len(tseq)
    left = _side(st, rev, q4, tseq, seq_len, table, a, b, jump_min_match, True)
    act, l, off, off2, _ = left
    clip = st[2] if not rev else qlen - st[3]
    if act == 2:
        third = ((st[5] >> 4) - l) << 4
        if st[4] == 1:
            st[6] = third
        st[5] = (clip + l) << 4
        st[4] += 2
        st[0] = off2 - (clip + l)
        if not rev:
            st[2] = 0
        else:
            st[3] = qlen
    elif act == 1:
        st[5] -= l << 4
        if st[4] == 1:
            st[6] = st[5]
        st[0] += l
        if not rev:
            st[2] += l
        else:
            st[3] -= l
    right = _side(st, rev, q4, tseq, seq_len, table, a, b, jump_min_match, False)
    return left, right
