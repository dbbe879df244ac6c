/* The DEFLATE entry points seen from plain C: they link, and without a context they fail before touching memory. */
#include <stdio.h>
#include <string.h>

#include "pixo_b200.h"

int main(void)
{
    const uint8_t data[4] = {1, 2, 3, 4};
    uint8_t out[64];
    size_t out_len = 0, lens[1] = {4}, out_lens[1] = {0};
    int32_t status[1] = {0};
    if (pixo_b200_deflate_zlib(NULL, data, sizeof data, 6, out, sizeof out, &out_len) != PIXO_B200_ERR_INVALID_ARGUMENT)
        return 1;
    if (!strstr(pixo_b200_last_error(NULL), "null context")) return 2;
    if (pixo_b200_deflate_zlib_on_device(NULL, data, 4, lens, 1, 6, out, sizeof out, out_lens, status) !=
        PIXO_B200_ERR_INVALID_ARGUMENT)
        return 3;
    if (PIXO_B200_ERR_INVALID_COMPRESSION_LEVEL != 14) return 4;
    printf("deflate_client ok\n");
    return 0;
}
