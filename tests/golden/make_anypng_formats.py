"""Writes tests/golden/anypng_formats: PNGs that PIL and OpenCV write in the formats the all-formats decode reads -- PIL palette
files at 1/2/4/8 bits with and without transparency, PIL mode "1" and "I;16" files, and cv2.imwrite 16-bit gray, BGR and BGRA
files -- from seeded random images, plus manifest.json.  The GPU test reads each file back with tests/pngwrite_formats.py's reader
and model.  Run from the repository root: python tests/golden/make_anypng_formats.py"""
import io
import json
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "anypng_formats")


def main():
    import cv2
    from PIL import Image
    os.makedirs(OUT, exist_ok=True)
    rs = np.random.RandomState(2024)
    manifest = []

    def save(name, data, writer):
        with open(os.path.join(OUT, name), "wb") as f:
            f.write(data)
        manifest.append({"file": name, "writer": writer})

    for bits in (1, 2, 4, 8):
        w, h = int(rs.randint(20, 60)), int(rs.randint(10, 40))
        im = Image.fromarray(rs.randint(0, 1 << bits, (h, w)).astype(np.uint8), "P")
        im.putpalette(rs.randint(0, 256, 3 * (1 << bits)).astype(np.uint8).tobytes())
        for tr in (False, True):
            b = io.BytesIO()
            extra = {"transparency": bytes(rs.randint(0, 256, 1 << bits).astype(np.uint8))} if tr else {}
            im.save(b, "PNG", bits=bits, **extra)
            save(f"pil_p{bits}{'_trns' if tr else ''}.png", b.getvalue(), "PIL")
    b = io.BytesIO()
    Image.fromarray((rs.randint(0, 2, (27, 45)) * 255).astype(np.uint8)).convert("1").save(b, "PNG")
    save("pil_mode1.png", b.getvalue(), "PIL")
    b = io.BytesIO()
    Image.fromarray(rs.randint(0, 65536, (31, 23)).astype(np.uint16)).save(b, "PNG")
    save("pil_i16.png", b.getvalue(), "PIL")
    for c in (1, 3, 4):
        img = rs.randint(0, 65536, (29, 41, c)).astype(np.uint16)
        ok, enc = cv2.imencode(".png", img if c > 1 else img[..., 0])
        assert ok
        save(f"cv2_u16_c{c}.png", enc.tobytes(), "OpenCV")
    with open(os.path.join(OUT, "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
