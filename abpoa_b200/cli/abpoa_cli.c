/* abpoa_cli.c -- the `abpoa` command line over libabpoa_b200 (reference src/abpoa.c:22-250: same options,
 * same output text).  A single input file runs one progressive MSA through abpoa_msa1; list mode (-l: one
 * FASTA/FASTQ file per line = one read group per line) is exactly the batched shape the GPU wants, so all
 * files are read first and go through ONE abpoa_gpu_msa_batch_write call; the output is what the reference
 * prints file by file.  Options whose subsystems are outside the hot-path scope (-S/-p seeding, -i restore,
 * -g plot, -d>1, -a1, -L) are accepted and then refused by the library with a message. */
#include <getopt.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "abpoa.h"
#include "abpoa_gpu.h"

#define CLI_VERSION "1.5.6-b200"

static const struct option long_opt[] = {
    { "align-mode", 1, NULL, 'm' }, { "match", 1, NULL, 'M' }, { "mismatch", 1, NULL, 'X' }, { "matrix", 1, NULL, 't' },
    { "gap-open", 1, NULL, 'O' }, { "gap-ext", 1, NULL, 'E' }, { "extra-b", 1, NULL, 'b' }, { "extra-f", 1, NULL, 'f' },
    { "zdrop", 1, NULL, 'z' }, { "bonus", 1, NULL, 'e' }, { "seeding", 0, NULL, 'S' }, { "k-mer", 1, NULL, 'k' },
    { "window", 1, NULL, 'w' }, { "min-poa-win", 1, NULL, 'n' }, { "progressive", 0, NULL, 'p' }, { "inc-path-score", 0, NULL, 'G' },
    { "sort-by-len", 0, NULL, 'L' }, { "gap-on-right", 0, NULL, 'R' }, { "gap-at-end", 0, NULL, 'J' }, { "use-qual-weight", 0, NULL, 'Q' },
    { "amino-acid", 0, NULL, 'c' }, { "in-list", 0, NULL, 'l' }, { "increment", 1, NULL, 'i' }, { "amb-strand", 0, NULL, 's' },
    { "output", 1, NULL, 'o' }, { "result", 1, NULL, 'r' }, { "out-pog", 1, NULL, 'g' }, { "cons-algrm", 1, NULL, 'a' },
    { "maxnum-cons", 1, NULL, 'd' }, { "min-freq", 1, NULL, 'q' }, { "help", 0, NULL, 'h' }, { "version", 0, NULL, 'v' },
    { "verbose", 1, NULL, 'V' }, { 0, 0, 0, 0 }
};

static int usage(void) {
    fprintf(stderr,
        "\nabpoa (GPU): adaptive banded Partial Order Alignment, DP on the GPU (libabpoa_b200 %s)\n\n"
        "Usage: abpoa [options] <in.fa/fq> > cons.fa / msa.fa\n\n"
        "  -m --align-mode INT   0: global, 1: local, 2: extension [0]\n"
        "  -M --match INT / -X --mismatch INT / -t --matrix FILE   scores [2 / 4 / none]\n"
        "  -O --gap-open INT(,INT) / -E --gap-ext INT(,INT)        gap penalties [4,24 / 2,1]\n"
        "  -b --extra-b INT / -f --extra-f FLOAT   adaptive band: w = b + f * L [10 / 0.01] (b < 0: no band)\n"
        "  -z --zdrop INT   -G --inc-path-score   -R --gap-on-right   -J --gap-at-end   -s --amb-strand\n"
        "  -Q --use-qual-weight   -c --amino-acid\n"
        "  -l --in-list          the input is a list of files, one read group per file (all groups run as one GPU batch)\n"
        "  -o --output FILE      [stdout]\n"
        "  -r --result INT       0: consensus FASTA, 1: RC-MSA, 2: both, 3: GFA, 4: GFA with consensus path,\n"
        "                        5: consensus FASTQ [0]\n"
        "  -h --help  -v --version  -V --verbose INT\n\n", CLI_VERSION);
    return 1;
}

/* one read group from a file: names, encoded reads, quality weights */
typedef struct { int n; char **names; int *lens; uint8_t **seqs; int **weights; } cli_group;

static double now_s(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + ts.tv_nsec * 1e-9; }

int main(int argc, char **argv) {
    int c, m, in_list = 0; char *s;
    abpoa_para_t *abpt = abpoa_init_para();
    while ((c = getopt_long(argc, argv, "m:M:X:t:O:E:b:f:z:e:GLRJQSk:w:n:i:clpso:r:g:a:d:q:hvV:", long_opt, NULL)) >= 0) {
        switch (c) {
        case 'm': m = atoi(optarg);
                  if (m != ABPOA_GLOBAL_MODE && m != ABPOA_EXTEND_MODE && m != ABPOA_LOCAL_MODE) { fprintf(stderr, "Unknown alignment mode: %d.\n", m); return 1; }
                  abpt->align_mode = m; break;
        case 'M': abpt->match = atoi(optarg); break;
        case 'X': abpt->mismatch = atoi(optarg); break;
        case 't': abpt->use_score_matrix = 1; abpt->mat_fn = strdup(optarg); break;
        case 'O': abpt->gap_open1 = (int)strtol(optarg, &s, 10); abpt->gap_open2 = *s == ',' ? (int)strtol(s + 1, &s, 10) : 0; break;
        case 'E': abpt->gap_ext1 = (int)strtol(optarg, &s, 10); abpt->gap_ext2 = *s == ',' ? (int)strtol(s + 1, &s, 10) : 0; break;
        case 'G': abpt->inc_path_score = 1; break;
        case 'L': abpt->sort_input_seq = 1; break;
        case 'R': abpt->put_gap_on_right = 1; break;
        case 'J': abpt->put_gap_at_end = 1; break;
        case 'b': abpt->wb = atoi(optarg); break;
        case 'f': abpt->wf = (float)atof(optarg); break;
        case 'z': abpt->zdrop = atoi(optarg); break;
        case 'e': abpt->end_bonus = atoi(optarg); break;
        case 'Q': abpt->use_qv = 1; break;
        case 'S': abpt->disable_seeding = 0; break;
        case 'k': abpt->k = atoi(optarg); break;
        case 'w': abpt->w = atoi(optarg); break;
        case 'n': abpt->min_w = atoi(optarg); break;
        case 'c': abpt->m = 27; abpt->mat = (int *)realloc(abpt->mat, (size_t)abpt->m * abpt->m * sizeof(int)); break;
        case 'i': abpt->incr_fn = strdup(optarg); break;
        case 'l': in_list = 1; break;
        case 'p': abpt->progressive_poa = 1; break;
        case 's': abpt->amb_strand = 1; break;
        case 'o': if (strcmp(optarg, "-") != 0 && freopen(optarg, "wb", stdout) == NULL) { fprintf(stderr, "Failed to open the output file %s\n", optarg); return 1; } break;
        case 'r': { const int r = atoi(optarg);
                  if (r == ABPOA_OUT_CONS) abpt->out_cons = 1, abpt->out_msa = 0;
                  else if (r == ABPOA_OUT_MSA) abpt->out_cons = 0, abpt->out_msa = 1;
                  else if (r == ABPOA_OUT_CONS_MSA) abpt->out_cons = abpt->out_msa = 1;
                  else if (r == ABPOA_OUT_GFA) abpt->out_cons = 0, abpt->out_gfa = 1;
                  else if (r == ABPOA_OUT_CONS_GFA) abpt->out_cons = 1, abpt->out_gfa = 1;
                  else if (r == ABPOA_OUT_CONS_FQ) abpt->out_cons = 1, abpt->out_fq = 1;
                  else fprintf(stderr, "Error: unknown output result mode: %s.\n", optarg);
                  break; }
        case 'g': abpt->out_pog = strdup(optarg); break;
        case 'a': abpt->cons_algrm = atoi(optarg); break;
        case 'd': abpt->max_n_cons = atoi(optarg);
                  if (abpt->max_n_cons < 1 || abpt->max_n_cons > 10) { fprintf(stderr, "Error: max number of consensus sequences should be 1~10.\n"); return 1; }
                  break;
        case 'q': abpt->min_freq = atof(optarg); break;
        case 'h': return usage();
        case 'V': abpt->verbose = atoi(optarg); break;
        case 'v': printf("%s\n", CLI_VERSION); abpoa_free_para(abpt); return 0;
        default:  fprintf(stderr, "Error: unknown option.\n"); return usage();
        }
    }
    if (argc - optind != 1) return usage();
    abpoa_post_set_para(abpt);
    fprintf(stderr, "[%s] CMD: ", "abpoa_b200");
    for (c = 0; c < argc; ++c) fprintf(stderr, " %s", argv[c]);
    fprintf(stderr, "\n");
    const double t0 = now_s();

    if (!in_list) {
        abpoa_t *ab = abpoa_init();
        abpoa_msa1(ab, abpt, argv[optind], stdout);
        abpoa_free(ab);
    } else {
        extern int poa_read_fastx(const char *fn, abpoa_seq_t *abs);
        extern void poa_encode_residues(const char *s, int l, uint8_t *out);
        FILE *lf = fopen(argv[optind], "r");
        if (!lf) { fprintf(stderr, "Failed to open the list file %s\n", argv[optind]); return 1; }
        int n_groups = 0, cap = 0; cli_group *gr = NULL;
        char fn[4096];
        abpoa_t *reader = abpoa_init();                      /* only its read container is used */
        while (fgets(fn, sizeof fn, lf)) {
            size_t l = strlen(fn);
            while (l > 0 && (fn[l - 1] == '\n' || fn[l - 1] == '\r')) fn[--l] = 0;
            if (l == 0) continue;
            if (n_groups == cap) { cap = cap ? cap * 2 : 64; gr = (cli_group *)realloc(gr, (size_t)cap * sizeof *gr); }
            cli_group *g = &gr[n_groups++];
            abpoa_seq_t *abs = reader->abs;
            abs->n_seq = 0;
            const int n = poa_read_fastx(fn, abs);
            if (n < 0) { fprintf(stderr, "fail to open file '%s'\n", fn); return 1; }
            g->n = n;
            g->names = (char **)calloc((size_t)(n > 0 ? n : 1), sizeof(char *)); g->lens = (int *)calloc((size_t)(n > 0 ? n : 1), sizeof(int));
            g->seqs = (uint8_t **)calloc((size_t)(n > 0 ? n : 1), sizeof(uint8_t *)); g->weights = (int **)calloc((size_t)(n > 0 ? n : 1), sizeof(int *));
            for (int i = 0; i < n; ++i) {
                const int sl = abs->seq[i].l;
                g->names[i] = strdup(abs->name[i].l > 0 ? abs->name[i].s : "");
                g->lens[i] = sl;
                g->seqs[i] = (uint8_t *)malloc((size_t)(sl > 0 ? sl : 1));
                poa_encode_residues(abs->seq[i].s, sl, g->seqs[i]);
                if (abpt->use_qv && abs->qual[i].l > 0) {
                    g->weights[i] = (int *)malloc((size_t)(sl > 0 ? sl : 1) * sizeof(int));
                    for (int j = 0; j < sl; ++j) g->weights[i][j] = (int)abs->qual[i].s[j] - 32;
                }
            }
        }
        fclose(lf);
        abpoa_free(reader);
        abpoa_gpu_group_t *groups = (abpoa_gpu_group_t *)calloc((size_t)(n_groups > 0 ? n_groups : 1), sizeof *groups);
        const char *const **names = (const char *const **)calloc((size_t)(n_groups > 0 ? n_groups : 1), sizeof *names);
        for (int g = 0; g < n_groups; ++g) {
            groups[g].n_seq = gr[g].n; groups[g].seq_lens = gr[g].lens; groups[g].seqs = (const uint8_t *const *)gr[g].seqs;
            groups[g].qual_weights = abpt->use_qv ? (const int *const *)gr[g].weights : NULL;
            names[g] = (const char *const *)gr[g].names;
        }
        if (n_groups > 0) {
            abpoa_gpu_batch_t *eng = abpoa_gpu_batch_init(-1, 0, 0);
            abpoa_gpu_msa_batch_write(eng, abpt, n_groups, groups, names, stdout, NULL, 0);
            abpoa_gpu_batch_free(eng);
        }
        for (int g = 0; g < n_groups; ++g) {
            for (int i = 0; i < gr[g].n; ++i) { free(gr[g].names[i]); free(gr[g].seqs[i]); free(gr[g].weights[i]); }
            free(gr[g].names); free(gr[g].lens); free(gr[g].seqs); free(gr[g].weights);
        }
        free(gr); free(groups); free((void *)names);
    }
    fprintf(stderr, "[abpoa_b200] Real time: %.3f sec.\n", now_s() - t0);
    abpoa_free_para(abpt);
    return 0;
}
