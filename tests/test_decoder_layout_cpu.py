"""CPU: numpy model of the shared-memory layouts and GMMA descriptor arithmetic of dec_conv7_tc_kernel
(neurad-studio_b200/csrc/rgb_decoder.cuh).  wgmma cannot run here, but the address arithmetic can: the model reads
the A / B operands through the canonical K-major no-swizzle descriptor rule
    element (row, k) of a bf16 operand = start + (row/8)*SBO + (k/8)*LBO + (row%8)*16 + (k%8)*2   [bytes]
exactly as the kernel programs them (plane-shifted activation windows, tap-column weight images with the tiles of one
column in descending dy so that up to three taps form one N = 96 operand), accumulates the same MMA sequence, and must reproduce torch's conv2d.  Integer-valued data keeps every product exact."""
import numpy as np
import torch
import torch.nn.functional as F

C, K7, PAD, STRIP, TH = 32, 7, 3, 128, 4
PW, IR = STRIP + 2 * PAD, TH + 2 * PAD
PLANE = (IR * PW * 16 + 127) // 128 * 128
WTILE = C * C * 2
WROW = K7 * 2 * WTILE


def fold_image(w):
    """dec_fold_conv_kernel's w_img (hi tiles only; lo tiles stay zero for integer weights)."""
    img = np.zeros(K7 * WROW, dtype=np.uint8)
    view = img.view(np.uint16)
    wb = (w.float().numpy().view(np.uint32) >> 16).astype(np.uint16)  # exact bf16 of small integers
    for co in range(C):
        for ci in range(C):
            for tap in range(K7 * K7):
                off = (co >> 3) * 512 + (ci >> 3) * 128 + (co & 7) * 16 + (ci & 7) * 2
                dy, dx = tap // K7, tap % K7
                view[(dx * WROW + (K7 - 1 - dy) * WTILE + off) // 2] = wb[co, ci, dy, dx]
    return img


def bf16_at(buf, byte_off):
    v = buf.view(np.uint16)[byte_off // 2].astype(np.uint32) << 16
    return v.view(np.float32)


def operand(buf, start, lbo, sbo, rows):
    """[rows,16] fp32 matrix the tensor core reads for one K=16 MMA."""
    r = np.arange(rows)[:, None]
    k = np.arange(16)[None, :]
    off = start + (r // 8) * sbo + (k // 8) * lbo + (r % 8) * 16 + (k % 8) * 2
    return bf16_at(buf, off)


def test_conv7_descriptor_walk_reproduces_conv2d():
    g = torch.Generator().manual_seed(0)
    H, W = 6, 20
    x = torch.randint(-3, 4, (1, C, H, W), generator=g).float()
    w = torch.randint(-2, 3, (C, C, K7, K7), generator=g).float()
    ref = F.conv2d(x, w, padding=PAD)[0].permute(1, 2, 0).numpy()  # [H,W,C]
    w_img = fold_image(w)
    xb = (x[0].permute(1, 2, 0).contiguous().numpy().view(np.uint32) >> 16).astype(np.uint16)  # [H,W,C] bf16 (hi)
    for y0 in range(0, H, TH):
        act = np.zeros(8 * PLANE, dtype=np.uint8)
        av = act.view(np.uint16)
        for ir in range(IR):
            for ip in range(PW):
                y, xx = y0 - PAD + ir, 0 - PAD + ip
                if 0 <= y < H and 0 <= xx < W:
                    for c in range(4):  # hi chunks; lo planes (4..7) stay zero
                        base = (c * PLANE + (ir * PW + ip) * 16) // 2
                        av[base:base + 8] = xb[y, xx, 8 * c:8 * c + 8]
        d = np.zeros((STRIP, TH * C), dtype=np.float64)  # [D0 | D1 | D2] side by side, as in TMEM
        for dx in range(K7):
            wcol = w_img[dx * WROW:(dx + 1) * WROW]
            for i in range(IR):  # input row i feeds output rows r_min..r_max through taps dy = i - r
                r_min, r_max = max(0, i - (K7 - 1)), min(TH - 1, i)
                nr = r_max - r_min + 1
                slot = (K7 - 1) - (i - r_min)
                for ks in range(2):
                    a = operand(act, 2 * ks * PLANE + (i * PW + dx) * 16, PLANE, 128, STRIP)
                    b = operand(wcol, slot * WTILE + ks * 256, 128, 512, C * nr)  # N = 32 * nr: concatenated tap tiles
                    d[:, r_min * C:(r_max + 1) * C] += a.astype(np.float64) @ b.astype(np.float64).T
        for r in range(TH):
            if y0 + r < H:
                assert np.array_equal(d[:W, r * C:(r + 1) * C], ref[y0 + r].astype(np.float64)), (y0, r)
