// ht2_gunzipsim.cpp -- TEST-ONLY host build of the chunked gzip inflate (ht2_inflate.h): the block finder, the
// speculative chunk decoder, the window propagation and the marker replacement run as host loops over the same source
// the device kernels use.
//
//   ht2_gunzipsim <in.gz> <out> <chunk_bytes>
//       inflates in.gz into out; prints the stats as one line of "key=value" pairs.  Exit 1 with the message on
//       stderr when the input is not valid gzip (nothing is written to out).
#include <stdio.h>
#include <stdlib.h>

#include "../../hisat2_b200/csrc/ht2_inflate.h"

int main(int argc, char** argv)
{
    if (argc != 4) { fprintf(stderr, "usage: ht2_gunzipsim <in.gz> <out> <chunk_bytes>\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { fprintf(stderr, "cannot open %s\n", argv[1]); return 2; }
    std::vector<uint8_t> in;
    uint8_t buf[1 << 16];
    size_t k;
    while ((k = fread(buf, 1, sizeof(buf), f)) > 0) in.insert(in.end(), buf, buf + k);
    fclose(f);
    Ht2zHostBackend be;
    ht2gpu_gunzip_stats_t S;
    memset(&S, 0, sizeof(S));
    std::string err;
    char* out = NULL;
    size_t len = 0;
    const int rc = ht2z_gunzip(be, in.data(), in.size(), (uint32_t)strtoul(argv[3], NULL, 10), &out, &len, S, err);
    if (rc != HT2GPU_OK) { fprintf(stderr, "gunzip: %s\n", err.c_str()); return 1; }
    FILE* o = fopen(argv[2], "wb");
    if (!o || fwrite(out, 1, len, o) != len || fclose(o) != 0) { fprintf(stderr, "cannot write %s\n", argv[2]); return 2; }
    free(out);
    printf("members=%llu blocks=%llu chunks=%llu confirmed=%llu merged_no_candidate=%llu merged_false_positive=%llu "
           "windows=%llu rounds=%llu windows_cut=%llu chunk_bytes=%u out_bytes=%llu\n",
           (unsigned long long)S.members, (unsigned long long)S.blocks, (unsigned long long)S.chunks,
           (unsigned long long)S.chunks_confirmed, (unsigned long long)S.chunks_merged_no_candidate,
           (unsigned long long)S.chunks_merged_false_positive, (unsigned long long)S.windows,
           (unsigned long long)S.decode_rounds, (unsigned long long)S.windows_cut, S.chunk_bytes, (unsigned long long)S.out_bytes);
    return 0;
}
