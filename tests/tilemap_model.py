"""numpy restatement of the training block map (lwm_b200/csrc/attn_tiles.cu, include/lwm_b200.h:
lwm_attn_step_tilemap), and the brute-force per-element mask it is held against."""
import numpy as np

MASKED_LOGIT = np.float32(-1.0e30)
LOG2E = np.float32(1.4426950408889634)
ZERO, MASKED, OTHER = 0, 1, 2


def bias_masked(bias_vals):
    """the kernels' test: bias * log2(e) < kMaskedLogit, in fp32"""
    with np.errstate(over="ignore"):   # finfo.min * log2(e) is -inf in fp32, as on the GPU
        return (np.asarray(bias_vals, np.float32) * LOG2E) < MASKED_LOGIT


def step_tilemap(bias, seg, Sq, Sk, q_pos0, k_pos0, causal):
    """bias [B, >= k_pos0+Sk] float32 or None, seg [B, ...] int32 or None ->
    (fwd: B x n_qt lists of kt*2+mixed, bwd: B x n_kt lists of qt*2+mixed)"""
    B = (bias if bias is not None else seg).shape[0]
    n_qt, n_q64, n_kt = Sq // 128, Sq // 64, Sk // 128
    fwd, bwd = [], []
    for b in range(B):
        qs = []
        for i in range(n_q64):
            pos = q_pos0 + 64 * i + np.arange(64)
            sid = seg[b, pos] if seg is not None else np.zeros(64, np.int64)
            own = (pos >= k_pos0) & (pos < k_pos0 + Sk)
            if bias is not None:
                own &= np.where(own, bias[b, np.minimum(pos, bias.shape[1] - 1)] == 0, False)
            qs.append((int(sid.min()), int(sid.max()), bool(own.all())))
        ks = []
        for j in range(n_kt):
            pos = k_pos0 + 128 * j + np.arange(128)
            sid = seg[b, pos] if seg is not None else np.zeros(128, np.int64)
            if bias is None:
                cls = ZERO
            else:
                bv = bias[b, pos]
                cls = ZERO if (bv == 0).all() else MASKED if bias_masked(bv).all() else OTHER
            ks.append((int(sid.min()), int(sid.max()), cls))

        def classify(q, k):
            if k[2] == MASKED or (seg is not None and (q[1] < k[0] or k[1] < q[0])):
                return 0
            if k[2] == ZERO and (seg is None or q[0] == q[1] == k[0] == k[1]):
                return 1
            return 2

        fl = []
        for t in range(n_qt):
            a, c = qs[2 * t], qs[2 * t + 1]
            q = (min(a[0], c[0]), max(a[1], c[1]), a[2] and c[2])
            n_vis = n_kt
            if causal:
                vis = q_pos0 + 128 * t + 127 - k_pos0
                n_vis = 0 if vis < 0 else min(n_kt, vis // 128 + 1)
            lst = []
            for kt in range(n_vis):
                cls = classify(q, ks[kt]) if q[2] else 2
                if cls:
                    lst.append(kt * 2 + (cls == 2))
            fl.append(lst)
        bl = []
        for kt in range(n_kt):
            i_start = 0
            if causal:
                diff = k_pos0 + 128 * kt - q_pos0
                i_start = 0 if diff <= 0 else min(diff // 64, n_q64)
            lst = []
            for qi in range(i_start, n_q64):
                cls = classify(qs[qi], ks[kt])
                if cls:
                    lst.append(qi * 2 + (cls == 2))
            bl.append(lst)
        fwd.append(fl)
        bwd.append(bl)
    return fwd, bwd


def element_masks(bias, seg, b, qpos, kpos, causal):
    """(full mask, causal-only mask) of rows qpos x keys kpos, True = masked, as the tile kernels evaluate them"""
    qpos, kpos = np.asarray(qpos)[:, None], np.asarray(kpos)[None, :]
    cm = (kpos > qpos) if causal else np.zeros((qpos.shape[0], kpos.shape[1]), bool)
    m = cm.copy()
    if bias is not None:
        m |= bias_masked(bias[b, kpos])
    if seg is not None:
        m |= seg[b, qpos] != seg[b, kpos]
    return m, cm


def row_proven(bias, b, pos, k_pos0, Sk):
    own = k_pos0 <= pos < k_pos0 + Sk
    return own and (bias is None or bias[b, pos] == 0)


def _packed(lengths, G, ids=None):
    seg = np.zeros(G, np.int32)
    p = 0
    for i, n in enumerate(lengths):
        seg[p:p + n] = i if ids is None else ids[i]
        p += n
    seg[p:] = len(lengths) if ids is None else ids[-1]
    return seg


def sweep_cases(B=2):
    """(name, bias [B,G] f32 or None, seg [B,G] i32 or None, Sq, Sk, q_pos0, k_pos0, causal)"""
    G = 1024
    rng = np.random.default_rng(7)
    fmin = np.finfo(np.float32).min
    cases = []
    # packed documents: boundaries on and off the 128 grid, documents of length 1
    docs = np.stack([_packed([128, 300, 1, 1, 84, 254, 128], G), _packed([1, 511, 1, 256, 7], G)])
    # non-monotone ids (a later document reuses an earlier id) and a single segment
    nonmono = np.stack([_packed([200, 300, 200], G, ids=[3, 1, 3, 0]), _packed([64, 700], G, ids=[5, 2, 5])])
    single = np.full((B, G), 7, np.int32)
    # bias: +-0, finfo.min and other finite values
    bias = np.zeros((B, G), np.float32)
    bias[0, 5:300] = -0.0
    bias[0, 384:640] = fmin
    bias[0, 700] = -1.5
    bias[1, :128] = fmin
    bias[1, 129:255] = fmin              # tile 1 has one visible key
    bias[1, 300:310] = 2.0
    bias[1, 512:768] = -1e30             # below the masked level after * log2(e)
    bias[1, 768:1024] = -6e29            # above it: finite, not masked
    pad = np.zeros((B, G), np.float32)   # left padding: 25 % off grid, 50 % on grid
    pad[0, :300] = fmin
    pad[1, :512] = fmin
    zseg = np.zeros((B, G), np.int32)
    for causal in (True, False):
        for q0, k0, Sq, Sk in ((0, 0, G, G), (512, 0, 512, 1024), (0, 256, 768, 512), (384, 640, 256, 384),
                               (0, 512, 512, 512)):
            c = "c" if causal else "nc"
            cases += [
                ("docs-%s-%d-%d" % (c, q0, k0), None, docs, Sq, Sk, q0, k0, causal),
                ("nonmono-%s-%d-%d" % (c, q0, k0), None, nonmono, Sq, Sk, q0, k0, causal),
                ("single-%s-%d-%d" % (c, q0, k0), None, single, Sq, Sk, q0, k0, causal),
                ("bias-%s-%d-%d" % (c, q0, k0), bias, None, Sq, Sk, q0, k0, causal),
                ("bias+docs-%s-%d-%d" % (c, q0, k0), bias, docs, Sq, Sk, q0, k0, causal),
                ("leftpad-%s-%d-%d" % (c, q0, k0), pad, zseg, Sq, Sk, q0, k0, causal),
                ("leftpad-biasonly-%s-%d-%d" % (c, q0, k0), pad, None, Sq, Sk, q0, k0, causal),
            ]
    rand_seg = np.sort(rng.integers(0, 9, (B, G)), axis=1).astype(np.int32)
    cases.append(("random-docs", None, rand_seg, G, G, 0, 0, True))
    return cases
