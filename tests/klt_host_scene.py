"""The frames rpg_svo_b200/host/host_klt_demo.cpp builds, restated: 752 x 480, frame k = a 7 x 7 box blur (integer
division) of an integer hash texture shifted by (3k, 2k) px, contrast stretched from [100, 155] to [0, 255].  Both sides use 32-bit unsigned wrap-around arithmetic."""
import numpy as np

W, H, N_FRAMES, N_LEVELS = 752, 480, 4, 5


def scene():
    yy, xx = np.mgrid[-3:H + 3 + 2 * N_FRAMES, -3:W + 3 + 3 * N_FRAMES].astype(np.int64)
    base = ((((xx & 0xFFFFFFFF) * 73856093) & 0xFFFFFFFF) ^ (((yy & 0xFFFFFFFF) * 19349663) & 0xFFFFFFFF)) >> 8 & 255
    imgs = []
    for k in range(N_FRAMES):
        s = np.zeros((H, W), np.int64)
        for j in range(7):
            for i in range(7):
                s += base[2 * k + j:2 * k + j + H, 3 * k + i:3 * k + i + W]
        v = np.clip(s // 49, 100, 155) - 100  # contrast stretched from [100, 155] to [0, 255]
        imgs.append((v * 255 // 55).astype(np.uint8))
    return imgs, N_LEVELS
