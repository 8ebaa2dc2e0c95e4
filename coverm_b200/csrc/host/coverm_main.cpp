// `coverm` binary: contig / genome coverage from BAM files on an H100 (links libcoverm_b200.so).
#include "../../../include/coverm_b200_host.h"
int main(int argc, char** argv) { return cmbh_main(argc, argv); }
