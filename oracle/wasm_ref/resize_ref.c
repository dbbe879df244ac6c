/*
 * resize_ref.c — runs pixo's resizer and its f32 sine from the reference's own wasm artefact, with the
 * interpreter of wasm_ref.c (included unchanged; its main is renamed out of the way).  Test
 * infrastructure only: it produces tests/golden/resize/ and checks oracle/resize.c's sinf.
 *
 * usage:
 *   resize_ref <pixo_bg.wasm> resize <in.raw> <sw> <sh> <dw> <dh> <color_type> <algorithm> <out>
 *       resizeImage(retptr, ptr, len, sw, sh, dw, dh, color_type, algorithm) -> out
 *   resize_ref <pixo_bg.wasm> sinf <first_bits> <last_bits> <step> all|differ <out>
 *       the wasm's sinf on the f32 bit patterns first, first+step, .. <= last: (x, sin x) f32 pairs -> out;
 *       with `differ` only the pairs where it is not (float)sin((double)x)
 *   resize_ref <pixo_bg.wasm> check <first_bits> <last_bits>
 *       every f32 bit pattern in [first, last] (same sign): the wasm's sinf against oracle/resize.c's
 *       rz_sinf and against (float)sin((double)x); prints "checked N oracle_mismatches M libm_differences L"
 *
 * The wasm's sinf is the one function of type (f32) -> f32 that returns 0x3f576aa4 (0.841470957) at 1.0;
 * it is looked up that way, not by index, and the index is printed.
 */
#define main wasm_ref_main
#include "wasm_ref.c"
#undef main
#include "../resize.c"

static uint32_t sinf_index(void)
{
    uint32_t found = 0xffffffffu;
    for (uint32_t fi = nimports; fi < nfuncs; fi++) {
        FuncType *t = &types[funcs[fi].type];
        if (t->np != 1 || t->nr != 1 || t->p[0] != 0x7D || t->r[0] != 0x7D) continue;
        vstack[vsp++] = 0x3f800000u;
        exec(fi);
        if ((uint32_t)vstack[--vsp] == 0x3f576aa4u) {
            if (found != 0xffffffffu) DIE("two candidate sinf functions: %u and %u", found, fi);
            found = fi;
        }
    }
    if (found == 0xffffffffu) DIE("no (f32) -> f32 function returns sin(1)");
    return found;
}

static uint32_t wasm_sinf(uint32_t fi, uint32_t bits)
{
    vstack[vsp++] = bits;
    exec(fi);
    return (uint32_t)vstack[--vsp];
}

int main(int argc, char **argv)
{
    if (argc < 3) DIE("usage: resize_ref <pixo_bg.wasm> resize|sinf|check ...");
    load_module(argv[1]);
    vstack = malloc(sizeof(uint64_t) * STACK_SLOTS);
    if (!strcmp(argv[2], "resize")) {
        if (argc != 11) DIE("bad argument count");
        size_t len; uint8_t *in = read_file(argv[3], &len);
        uint32_t a1[1] = {(uint32_t)-16};
        uint32_t retptr = call_n("__wbindgen_add_to_stack_pointer", 1, a1, 1);
        uint32_t a2[2] = {(uint32_t)len, 1};
        uint32_t ptr0 = len ? call_n("__wbindgen_export", 2, a2, 1) : 1;
        mem_check(ptr0, (uint32_t)len); memcpy(mem + ptr0, in, len);
        uint32_t a[9] = {retptr, ptr0, (uint32_t)len};
        for (int i = 0; i < 6; i++) a[3 + i] = (uint32_t)strtoul(argv[4 + i], NULL, 10);
        call_n("resizeImage", 9, a, 0);
        uint32_t r[4]; mem_check(retptr, 16); memcpy(r, mem + retptr, 16);
        if (r[3]) { fprintf(stderr, "pixo error: %s\n", last_error); return 3; }
        mem_check(r[0], r[1]);
        FILE *fo = fopen(argv[10], "wb"); if (!fo) DIE("cannot write %s", argv[10]);
        fwrite(mem + r[0], 1, r[1], fo); fclose(fo);
        return 0;
    }
    const uint32_t fi = sinf_index();
    fprintf(stderr, "sinf is wasm function %u\n", fi);
    if (!strcmp(argv[2], "sinf")) {
        if (argc != 8) DIE("bad argument count");
        const int differ = !strcmp(argv[6], "differ");
        const uint32_t first = (uint32_t)strtoul(argv[3], NULL, 0), last = (uint32_t)strtoul(argv[4], NULL, 0);
        const uint32_t step = (uint32_t)strtoul(argv[5], NULL, 0);
        FILE *fo = fopen(argv[7], "wb"); if (!fo) DIE("cannot write %s", argv[7]);
        for (uint64_t b = first; b <= last; b += step) {
            uint32_t pair[2] = {(uint32_t)b, wasm_sinf(fi, (uint32_t)b)};
            float x, ref;
            memcpy(&x, &pair[0], 4);
            ref = (float)sin((double)x);
            if (!differ || memcmp(&ref, &pair[1], 4)) fwrite(pair, 4, 2, fo);
        }
        fclose(fo);
        return 0;
    }
    if (!strcmp(argv[2], "check")) {
        if (argc != 5) DIE("bad argument count");
        const uint32_t first = (uint32_t)strtoul(argv[3], NULL, 0), last = (uint32_t)strtoul(argv[4], NULL, 0);
        uint64_t n = 0, bad = 0, libm = 0;
        for (uint64_t b = first; b <= last; b++) {
            float x, want, ours, ref;
            uint32_t xb = (uint32_t)b, wb = wasm_sinf(fi, xb);
            memcpy(&x, &xb, 4); memcpy(&want, &wb, 4);
            ours = rz_sinf(x);
            ref = (float)sin((double)x);
            if (memcmp(&ours, &want, 4)) {
                if (bad < 20) fprintf(stderr, "mismatch at %08x: wasm %08x oracle %a\n", xb, wb, ours);
                bad++;
            }
            libm += memcmp(&ref, &want, 4) != 0;
            n++;
        }
        printf("checked %llu oracle_mismatches %llu libm_differences %llu\n", (unsigned long long)n,
               (unsigned long long)bad, (unsigned long long)libm);
        return bad != 0;
    }
    DIE("unknown mode %s", argv[2]);
}
