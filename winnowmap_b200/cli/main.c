/* winnowmap-b200: the winnowmap command line over the GPU mapper (wm_cli_main, include/winnowmap_b200.h) */
#include "winnowmap_b200.h"

int main(int argc, char *argv[])
{
	return wm_cli_main(argc, argv);
}
