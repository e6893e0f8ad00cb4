/* ssqo_main.c — ORACLE (test infrastructure): CLI with the argv contract of the reference's
 * `$BWA index|mem` and `$SAMBLASTER` call sites (speedseq/bin/speedseq:389,438-439). */
#include <string.h>
#include <stdio.h>
#include "ssqo.h"
extern const char *ssqo_prog;
int main(int argc, char **argv)
{
	const char *base = strrchr(argv[0], '/');
	base = base ? base + 1 : argv[0];
	ssqo_prog = argv[0];
	if (strstr(base, "samblaster")) return ssqo_main_samblaster(argc, argv);
	if (argc < 2) { fprintf(stderr, "Usage: %s <index|mem|samblaster> ...\n", argv[0]); return 1; }
	if (!strcmp(argv[1], "index")) return ssqo_main_index(argc - 1, argv + 1);
	if (!strcmp(argv[1], "mem")) return ssqo_main_mem(argc - 1, argv + 1);
	if (!strcmp(argv[1], "samblaster")) return ssqo_main_samblaster(argc - 1, argv + 1);
	fprintf(stderr, "[main] unrecognized command '%s'\n", argv[1]);
	return 1;
}
