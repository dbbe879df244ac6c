/* The whole-file PNG entry points seen from plain C: they link, and without a context they refuse bad input in pixo's
 * order before touching memory, then refuse the missing context. */
#include <stdio.h>
#include <string.h>

#include "pixo_b200.h"

int main(void)
{
    uint8_t data[4 * 4 * 4] = {0}, out[64];
    size_t out_len = 0, out_lens[1] = {0};
    int32_t status[1] = {0};
    const uint32_t fast = PIXO_B200_FILTER_ADAPTIVE_FAST;
    if (pixo_b200_png_encode(NULL, data, sizeof data, 4, 4, PIXO_B200_RGBA, fast, 0, 256, NULL, 0, out, sizeof out,
                             &out_len) != PIXO_B200_ERR_INVALID_COMPRESSION_LEVEL)
        return 1;
    if (pixo_b200_png_encode(NULL, data, sizeof data, 0, 4, PIXO_B200_RGBA, fast, 2, 256, NULL, 0, out, sizeof out,
                             &out_len) != PIXO_B200_ERR_INVALID_DIMENSIONS)
        return 2;
    if (pixo_b200_png_encode(NULL, data, sizeof data, 4, 4, PIXO_B200_RGBA, fast | PIXO_B200_PNG_OPTIMAL_COMPRESSION,
                             9, 256, NULL, 0, out, sizeof out, &out_len) != PIXO_B200_ERR_UNSUPPORTED)
        return 3;
    if (!strstr(pixo_b200_last_error(NULL), "optimal_compression")) return 4;
    if (pixo_b200_png_encode(NULL, data, sizeof data, 4, 4, PIXO_B200_RGBA, fast, 2, 256, NULL, 0, out, sizeof out,
                             &out_len) != PIXO_B200_ERR_INVALID_ARGUMENT)
        return 5;
    if (!strstr(pixo_b200_last_error(NULL), "ctx is null")) return 6;
    if (pixo_b200_png_encode_on_device(NULL, data, sizeof data, 1, 4, 4, PIXO_B200_RGBA, fast, 6, 256, NULL, NULL, out,
                                       sizeof out, out_lens, status, NULL) != PIXO_B200_ERR_INVALID_ARGUMENT)
        return 7;
    printf("png_encode_client ok\n");
    return 0;
}
