"""numpy restatement of the reference's Embedding job (Embedding.scala:27-51, 53-101, 103-138): Spark MLlib's
`Word2Vec` (hierarchical-softmax skip-gram, SGD) over each user's positive ratings, and the user embeddings.

THIS IS THE READABLE SPEC, NOT PRODUCT.  Every float32 statement rounds once per operation, as the JVM does, and
the training loop runs one (centre word, context word) pair at a time, so it is slow: use it on short horizons.
`oracle/item2vec_c.c` (`item2vec_cext`) runs the same statements in plain C for full runs, and the tests hold the
two to each other bit for bit.  DESIGN.md section 4.12 gives the semantics and the orders Spark leaves open.
"""
from __future__ import annotations

import math

import numpy as np

MIN_COUNT = 5
LEARNING_RATE = 0.025
MAX_SENTENCE_LENGTH = 1000
MAX_EXP = 6
EXP_TABLE_SIZE = 1000
MAX_CODE_LENGTH = 40          # Spark's bound; the device supports 32
_M64 = (1 << 64) - 1
_GOLDEN = 0x9E3779B97F4A7C15
f32 = np.float32


# ---- sentences and vocabulary -----------------------------------------------------------------------------------

def ts_string_key(ts):
    """The timestamp's decimal string as a sortable integer: left-aligned to 10 digits, then the digit count (a
    string prefix sorts first).  featureeng.cu's sort key."""
    ts = np.asarray(ts, np.int64)
    digits = np.array([len(str(t)) for t in ts.tolist()], np.int64)
    return ts * 10 ** (10 - digits) * 16 + digits


def positive_sequences(user, movie, half, ts):
    """processItemSequence (Embedding.scala:27-51): positive ratings (half-stars >= 7) grouped by user, users
    ascending, each user's movies ordered by the timestamp string with ties in file order.  Returns (users [S],
    list of int64 arrays of movie ids)."""
    user, movie, half = (np.asarray(a, np.int64) for a in (user, movie, half))
    pos = np.flatnonzero(half >= 7)
    order = pos[np.lexsort((pos, ts_string_key(np.asarray(ts)[pos]), user[pos]))]
    u = user[order]
    starts = np.flatnonzero(np.r_[True, u[1:] != u[:-1]]) if len(u) else np.zeros(0, np.int64)
    bounds = np.r_[starts, len(u)]
    return u[starts], [movie[order[bounds[i]:bounds[i + 1]]] for i in range(len(starts))]


def build_vocab(seqs, min_count=MIN_COUNT):
    """Spark's learnVocab: count every word, keep count >= min_count, sort by count descending (ties: movie id
    ascending).  Returns (ids [V] int64, counts [V] int64)."""
    allw = np.concatenate(seqs) if seqs else np.zeros(0, np.int64)
    ids, cnt = np.unique(allw, return_counts=True)
    keep = cnt >= min_count
    ids, cnt = ids[keep], cnt[keep]
    o = np.lexsort((ids, -cnt))
    return ids[o], cnt[o].astype(np.int64)


def chunk_corpus(seqs, ids, max_len=MAX_SENTENCE_LENGTH):
    """Map each sentence to vocabulary indices, drop words outside the vocabulary, cut into chunks of max_len.
    Returns (words int32 [N], offsets int64 [S + 1])."""
    index = {int(m): i for i, m in enumerate(ids.tolist())}
    words, offs = [], [0]
    for s in seqs:
        w = [index[m] for m in s.tolist() if m in index]
        for c in range(0, len(w), max_len):
            words.extend(w[c:c + max_len])
            offs.append(len(words))
    return np.asarray(words, np.int32), np.asarray(offs, np.int64)


def huffman(counts):
    """createBinaryTree (word2vec.c's, as Spark restates it): internal nodes start at 1e9, the two smallest are
    merged with ties going to the internal node.  Returns (code [V][40] int8, point [V][40] int32, codelen [V])."""
    V = len(counts)
    count = np.zeros(2 * V + 1, np.int64)
    count[:V] = counts
    count[V:2 * V] = int(1e9)
    binary = np.zeros(2 * V + 1, np.int64)
    parent = np.zeros(2 * V + 1, np.int64)
    pos1, pos2 = V - 1, V
    for a in range(V - 1):
        mins = []
        for _ in range(2):
            if pos1 >= 0 and count[pos1] < count[pos2]:
                mins.append(pos1)
                pos1 -= 1
            else:
                mins.append(pos2)
                pos2 += 1
        count[V + a] = count[mins[0]] + count[mins[1]]
        parent[mins[0]] = parent[mins[1]] = V + a
        binary[mins[1]] = 1
    code = np.zeros((V, MAX_CODE_LENGTH), np.int8)
    point = np.zeros((V, MAX_CODE_LENGTH + 1), np.int32)
    codelen = np.zeros(V, np.int32)
    for a in range(V):
        b, cs, ps = a, [], []
        while b != 2 * V - 2:
            cs.append(binary[b])
            ps.append(b)
            b = parent[b]
        i = len(cs)
        if i > MAX_CODE_LENGTH:
            raise ValueError("word %d: Huffman code of length %d > %d" % (a, i, MAX_CODE_LENGTH))
        codelen[a] = i
        point[a, 0] = V - 2
        for k in range(i):
            code[a, i - k - 1] = cs[k]
            point[a, i - k] = ps[k] - V
    return code, point[:, :MAX_CODE_LENGTH], codelen


# ---- the fixed tables and the schedule -------------------------------------------------------------------------

def exp_table():
    """expTable[i] = (float)(t / (t + 1)), t = exp((2.0 i / 1000 - 1.0) * 6)."""
    t = [math.exp((2.0 * i / EXP_TABLE_SIZE - 1.0) * MAX_EXP) for i in range(EXP_TABLE_SIZE)]   # the C library's exp
    return np.array([x / (x + 1.0) for x in t], np.float64).astype(np.float32)


def exp_index(f):
    """((f + MAX_EXP) * (EXP_TABLE_SIZE / MAX_EXP / 2.0)).toInt: the float sum, then a double product with 83.0
    (Scala's integer 1000 / 6 = 166, halved)."""
    return int(float(f32(f) + f32(MAX_EXP)) * float(EXP_TABLE_SIZE // MAX_EXP / 2.0))


def alpha_at(lr, partitions, word_count, k, train_words, iterations):
    """The learning rate a partition sets at a sentence start once > 10 000 words went by since the last update:
    lr * (1 - (P * wordCount + (k - 1) * trainWordsCount) / (iterations * trainWordsCount + 1)), floored at
    lr * 1e-4.  All double."""
    a = lr * (1 - (partitions * float(word_count) + float((k - 1) * train_words))
              / float(iterations * train_words + 1))
    return max(a, lr * 0.0001)


# ---- the counter-based generator --------------------------------------------------------------------------------

def _mix(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def splitmix(x, i):
    """srs_fill_uniform's hash: splitmix64's finaliser of x + (i + 1) * golden (mod 2^64)."""
    return _mix((x + (i + 1) * _GOLDEN) & _M64)


def init_syn0(seed, V, D):
    """syn0 = (u - 0.5f) / vectorSize, u = the top 24 bits of splitmix(seed, element) / 2^24; float32."""
    seed &= _M64
    i = np.arange(V * D, dtype=np.uint64)
    z = np.uint64(seed) + (i + np.uint64(1)) * np.uint64(_GOLDEN)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    u = (z >> np.uint64(40)).astype(np.float32) * f32(1.0 / 16777216.0)
    return ((u - f32(0.5)) / f32(D)).astype(np.float32).reshape(V, D)


def window_b(seed, k, p, t, window):
    """`random.nextInt(window)` of iteration k (1-based), partition p, for the centre word at corpus position t:
    the high 32 bits of splitmix(splitmix(splitmix(~seed, k), p), t), modulo window."""
    r = splitmix(splitmix(splitmix(~seed & _M64, k), p), t)
    return (r >> 32) % window


# ---- training -----------------------------------------------------------------------------------------------------

def train_pair(s0, s1, last, word, code, point, codelen, alpha, exp, m1):
    """One (centre word, context word) pair: syn0[last] walks the centre word's Huffman path."""
    L = int(codelen[word])
    pts = point[word, :L]
    x0 = s0[last].copy()
    D = s0.shape[1]
    f = np.zeros(L, np.float32)
    for j in range(D):                                     # sdot: sequential over the dimensions, no FMA
        f = f + x0[j] * s1[pts, j]
    neu1e = np.zeros(D, np.float32)
    for d in range(L):
        if not (f[d] > -MAX_EXP and f[d] < MAX_EXP):
            continue
        e = exp[exp_index(f[d])]
        g = f32(float(f32(1 - int(code[word, d])) - e) * alpha)
        l2 = pts[d]
        neu1e = neu1e + g * s1[l2]                           # syn1 before its update
        s1[l2] = s1[l2] + g * x0
        m1[l2] = True
    s0[last] = s0[last] + neu1e


def train_partition(s0, s1, m0, m1, words, offs, sent_ids, k, p, P, seed, window, iterations, train_words, code,
                    point, codelen, exp, lr=LEARNING_RATE):
    alpha, wc, lwc = lr, 0, 0
    for i in sent_ids:
        if wc - lwc > 10000:
            lwc = wc
            alpha = alpha_at(lr, P, wc, k, train_words, iterations)
        lo, hi = int(offs[i]), int(offs[i + 1])
        sent = words[lo:hi]
        n = hi - lo
        wc += n
        for pos in range(n):
            word = int(sent[pos])
            b = window_b(seed, k, p, lo + pos, window)
            for a in range(b, 2 * window + 1 - b):
                if a == window:
                    continue
                c = pos - window + a
                if 0 <= c < n:
                    last = int(sent[c])
                    train_pair(s0, s1, last, word, code, point, codelen, alpha, exp, m1)
                    m0[last] = True


def merge(glob, local, modified):
    """End of an iteration: every row modified by one or more partitions becomes the sum of those partitions' rows
    in partition order, times 1.0f / count; other rows keep the global value."""
    out = glob.copy()
    for r in range(glob.shape[0]):
        parts = [p for p in range(len(local)) if modified[p][r]]
        if not parts:
            continue
        v = local[parts[0]][r].copy()
        for p in parts[1:]:
            v = v + local[p][r]
        out[r] = v * (f32(1.0) / f32(len(parts)))
    return out


def train(words, offs, counts, code, point, codelen, vector_size, window, iterations, partitions, seed,
          lr=LEARNING_RATE):
    """Word2Vec.fit's loop: returns syn0 [V][vector_size] float32."""
    V, D = len(counts), vector_size
    train_words = int(np.sum(counts))
    exp = exp_table()
    syn0 = init_syn0(seed, V, D)
    syn1 = np.zeros((V, D), np.float32)
    n_sent = len(offs) - 1
    for k in range(1, iterations + 1):
        l0, l1, m0, m1 = [], [], [], []
        for p in range(partitions):
            s0, s1 = syn0.copy(), syn1.copy()
            a0, a1 = np.zeros(V, bool), np.zeros(V, bool)
            train_partition(s0, s1, a0, a1, words, offs, range(p, n_sent, partitions), k, p, partitions, seed,
                            window, iterations, train_words, code, point, codelen, exp, lr)
            l0.append(s0); l1.append(s1); m0.append(a0); m1.append(a1)
        syn0, syn1 = merge(syn0, l0, m0), merge(syn1, l1, m1)
    return syn0


def item2vec(user, movie, half, ts, vector_size=10, window=5, iterations=10, partitions=1, seed=0):
    """ratings -> (vocabulary ids [V], vectors [V][vector_size]): the whole job, for short horizons."""
    _, seqs = positive_sequences(user, movie, half, ts)
    ids, counts = build_vocab(seqs)
    words, offs = chunk_corpus(seqs, ids)
    code, point, codelen = huffman(counts)
    return ids, train(words, offs, counts, code, point, codelen, vector_size, window, iterations, partitions, seed)


# ---- user embeddings ------------------------------------------------------------------------------------------------

def user_embeddings(user, movie, ids, vectors):
    """generateUserEmb as the shipped userEmb.csv was made: per user (ascending), the float32 sum of the vectors of
    all the user's rated movies that have one, in reverse file order (foldRight), no division; zero if none."""
    user, movie = np.asarray(user, np.int64), np.asarray(movie, np.int64)
    row = {int(m): i for i, m in enumerate(np.asarray(ids).tolist())}
    users = np.unique(user)
    out = np.zeros((len(users), vectors.shape[1]), np.float32)
    order = np.argsort(user, kind="stable")
    bounds = np.searchsorted(user[order], users, side="left").tolist() + [len(user)]
    for ui in range(len(users)):
        acc = np.zeros(vectors.shape[1], np.float32)
        for f in order[bounds[ui]:bounds[ui + 1]][::-1].tolist():
            r = row.get(int(movie[f]))
            if r is not None:
                acc = acc + vectors[r]
        out[ui] = acc
    return users.astype(np.int32), out
