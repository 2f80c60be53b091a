/* Scalar plain-C restatement of the breakout_pixels renderer (oracle/SPEC_BREAKOUT_PIXELS.md).
 * TEST INFRASTRUCTURE (see oracle/__init__.py): oracle/breakout_pixels.py steps the game with the breakout oracle of
 * envs.c and draws each frame here from the breakout observation row.  One frame pixel at a time, the max over its
 * field rectangle -- deliberately not shaped like the CUDA kernel.
 */
#include <stdint.h>

typedef struct {
    int px, bx, by;
    uint8_t bricks[120];
} Scene;

/* the value of field pixel (x, y), 0 <= x < 160, 0 <= y < 200 */
static int field_pixel(const Scene* s, int x, int y) {
    if (x >= s->bx && x < s->bx + 2 && y >= s->by && y < s->by + 2) return 255;
    if (x >= s->px && x < s->px + 24 && (y == 190 || y == 191)) return 192;
    if (y >= 30 && y < 66) {
        int row = (y - 30) / 6, col = x / 8;
        if (s->bricks[row * 20 + col]) return 176 - 16 * row;
    }
    return 0;
}

/* rows: n breakout observation rows of 128 floats ([px/256, bx/256, by/256, ..., brick_0 .. brick_119]);
 * frames: n frames of 84 x 84 bytes */
void oracle_breakout_pixels_render(const float* rows, int n, uint8_t* frames) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; i++) {
        const float* o = rows + (int64_t)i * 128;
        Scene s;
        s.px = (int)(o[0] * 256.0f);   /* k / 256 is exact in fp32 */
        s.bx = (int)(o[1] * 256.0f);
        s.by = (int)(o[2] * 256.0f);
        for (int b = 0; b < 120; b++) s.bricks[b] = o[8 + b] != 0.0f;
        uint8_t* f = frames + (int64_t)i * 84 * 84;
        for (int r = 0; r < 84; r++)
            for (int c = 0; c < 84; c++) {
                int v = 0;
                for (int y = 200 * r / 84; y < 200 * (r + 1) / 84; y++)
                    for (int x = 160 * c / 84; x < 160 * (c + 1) / 84; x++) {
                        int p = field_pixel(&s, x, y);
                        if (p > v) v = p;
                    }
                f[r * 84 + c] = (uint8_t)v;
            }
    }
}
